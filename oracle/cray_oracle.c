/*
 * cray_oracle.c — CPU restatement of c-ray's hot loop (see cray_oracle.h).  Plain C99, compiled with
 * -ffp-contract=off so every a*b+c rounds twice like the strict reference build.  Each function cites
 * the reference file:line it restates.  Written against the flat scene (include/crscene.h), not the
 * reference's structs; no reference source is included or linked.
 */
#include "cray_oracle.h"
#include <math.h>
#include <float.h>
#include <stdlib.h>
#include <string.h>
#include <stdbool.h>
#include <pthread.h>

#define PI 3.141592653589793238462643383279502f /* includes.h:13 */

typedef struct { float x, y, z; } v3;
typedef struct { float x, y; } v2;
typedef struct { float r, g, b, a; } col;

/* includes.h:20-21 — ternary macros; operand order and NaN behaviour matter */
#define MIN_(a, b) (((a) < (b)) ? (a) : (b))
#define MAX_(a, b) (((a) > (b)) ? (a) : (b))

/* ---- libm semantics ----------------------------------------------------------------------------------
 * Every libm call of the hot loop goes through lm_*().  Semantics 0 is the reference: glibc's fp32 routine.  Semantics 1 is the
 * device (crgpu_math.cuh): the fp64 function rounded once to fp32, powf as exp(y*log x) on its fast branch, and powf(x, 5) of
 * schlick() as fp64 products.  The device's fp64 routines are not glibc's (CUDA documents up to 2 ulp, glibc up to 1), so an fp64
 * result that lies within a few fp64 ulps of an fp32 rounding boundary may round the other way on the device: such an evaluation
 * sets the thread's near-tie flag (lm_tie), which the callers report per path.  The mode and the flag are per thread: every
 * worker sets lm_sem from its job and clears lm_tie per path. */
static _Thread_local int lm_sem;
static _Thread_local int lm_tie;
#define LM_TIE_ULPS 4.0   /* CUDA's error bound + glibc's, with a margin */

/* flags r when an fp32 rounding boundary (the midpoint between two adjacent floats; for subnormal results the absolute grid) lies
 * within LM_TIE_ULPS * scale fp64 ulps of it */
static void lm_check(double r, double scale) {
	if (!isfinite(r)) return;
	const double a = fabs(r);
	const float f = (float)r;
	double lo, hi;                                       /* the boundaries either side of f */
	const double top = (double)FLT_MAX + ldexp(1.0, 103);   /* FLT_MAX and +inf round apart here */
	if (isinf(f)) { lo = hi = signbit(f) ? -top : top; }
	else {
		const float fd = nextafterf(f, -INFINITY), fu = nextafterf(f, INFINITY);
		lo = isinf(fd) ? -top : ((double)f + (double)fd) * 0.5;
		hi = isinf(fu) ? top : ((double)f + (double)fu) * 0.5;
	}
	const double ulp = nextafter(a, INFINITY) - a;
	const double tol = LM_TIE_ULPS * scale * ulp;
	if (fabs(r - lo) <= tol || fabs(r - hi) <= tol) lm_tie = 1;
}
static inline float lm_round(double r, double scale) { lm_check(r, scale); return (float)r; }

static float lm_sinf(float x) { return lm_sem ? lm_round(sin((double)x), 1.0) : sinf(x); }
static float lm_cosf(float x) { return lm_sem ? lm_round(cos((double)x), 1.0) : cosf(x); }
static float lm_tanf(float x) { return lm_sem ? lm_round(tan((double)x), 1.0) : tanf(x); }
static float lm_logf(float x) { return lm_sem ? lm_round(log((double)x), 1.0) : logf(x); }
static float lm_log10f(float x) { return lm_sem ? lm_round(log10((double)x), 1.0) : log10f(x); }
static float lm_atan2f(float y, float x) { return lm_sem ? lm_round(atan2((double)y, (double)x), 1.0) : atan2f(y, x); }
static float lm_acosf(float x) { return lm_sem ? lm_round(acos((double)x), 1.0) : acosf(x); }
static float lm_asinf(float x) { return lm_sem ? lm_round(asin((double)x), 1.0) : asinf(x); }
/* cr_powf: exp(y*log x) on 0 < x < FLT_MAX, finite y, |y| < 1e6, where an error of the fp64 log is magnified |y ln x| times;
 * the full pow() special-case logic everywhere else */
static float lm_powf(float x, float y) {
	if (!lm_sem) return powf(x, y);
	if (x > 0.0f && x < FLT_MAX && y == y && fabsf(y) < 1.0e6f) {
		const double e = (double)y * log((double)x);
		return lm_round(exp(e), 1.0 + fabs(e));
	}
	return lm_round(pow((double)x, (double)y), 1.0);
}
/* powf(x, 5.0f) of schlick(); cr_pow5f is four exact-order fp64 products, which this restates operation for operation */
static float lm_pow5f(float x) {
	if (!lm_sem) return powf(x, 5.0f);
	const double a = (double)x, a2 = a * a;
	return (float)(a2 * a2 * a);
}

/* ---- vector.h ------------------------------------------------------------------------------------ */
static inline v3 v3add(v3 a, v3 b) { return (v3){ a.x + b.x, a.y + b.y, a.z + b.z }; }          /* :65 */
static inline v3 v3sub(v3 a, v3 b) { return (v3){ a.x - b.x, a.y - b.y, a.z - b.z }; }          /* :76 */
static inline v3 v3mul(v3 a, v3 b) { return (v3){ a.x * b.x, a.y * b.y, a.z * b.z }; }          /* :80 */
static inline float v3dot(v3 a, v3 b) { return a.x * b.x + a.y * b.y + a.z * b.z; }             /* :91 */
static inline v3 v3scale(v3 v, float c) { return (v3){ v.x * c, v.y * c, v.z * c }; }           /* :102 */
static inline v3 v3cross(v3 a, v3 b) {                                                          /* :121 */
	return (v3){ (a.y * b.z) - (a.z * b.y), (a.z * b.x) - (a.x * b.z), (a.x * b.y) - (a.y * b.x) };
}
static inline float v3len(v3 v) { return sqrtf(v3dot(v, v)); }                                  /* :162 */
static inline v3 v3norm(v3 v) { float l = v3len(v); return (v3){ v.x / l, v.y / l, v.z / l }; } /* :173 */
static inline v3 v3neg(v3 v) { return (v3){ -v.x, -v.y, -v.z }; }                               /* :200 */
static inline v3 v3reflect(v3 I, v3 N) { return v3sub(I, v3scale(N, v3dot(N, I) * 2.0f)); }     /* :211 */
static inline float clampf(float value, float lo, float hi) { return MIN_(MAX_(value, lo), hi); } /* :55 */
static inline float wrapMax(float x, float max) { return fmodf(max + fmodf(x, max), max); }     /* :215 */
static inline float wrapMinMax(float x, float min, float max) { return min + wrapMax(x - min, max - min); } /* :219 */

/* ---- color.h ------------------------------------------------------------------------------------- */
static inline col cmul(col a, col b) { return (col){ a.r * b.r, a.g * b.g, a.b * b.b, a.a * b.a }; }   /* :33 */
static inline col cadd(col a, col b) { return (col){ a.r + b.r, a.g + b.g, a.b + b.b, a.a + b.a }; }   /* :38 */
static inline col ccoef(float k, col c) { return (col){ c.r * k, c.g * k, c.b * k, c.a * k }; }        /* :49 */
static inline col cmix(col a, col b, float t) { return cadd(ccoef(1.0f - t, a), ccoef(t, b)); }        /* :54 */
static inline float srgb_to_linear(float c) {                                                           /* :68 */
	if (c <= 0.04045f) return c / 12.92f;
	return lm_powf(((c + 0.055f) / 1.055f), 2.4f);
}
static inline float linear_to_srgb(float c) {                                                           /* :60 */
	if (c <= 0.0031308f) return 12.92f * c;
	return (1.055f * lm_powf(c, 0.4166666667f)) - 0.055f;
}
static inline col to_grayscale(col c) {                                                                 /* :43 — note the double constants */
	float b = sqrtf(0.299f * lm_powf(c.r, 2) + 0.587 * lm_powf(c.g, 2) + 0.114 * lm_powf(c.b, 2));
	return (col){ b, b, b, c.a };
}
static col color_for_kelvin(float kelvin) {                                                             /* color.c:28-70 */
	col ret = { 0 };
	float temp = kelvin >= 40000.0f ? 40000.0f : kelvin;
	temp = temp / 100.0f;
	if (temp <= 66.0f) {
		ret.r = 255.0f;
	} else {
		ret.r = temp - 60.0f;
		ret.r = 329.698727446f * lm_powf(ret.r, -0.1332047592f);
		ret.r = ret.r < 0.0f ? 0.0f : ret.r;
		ret.r = ret.r > 255.0f ? 255.0f : ret.r;
	}
	if (temp <= 66.0f) {
		ret.g = temp;
		ret.g = 99.4708025861f * lm_logf(ret.g) - 161.1195681661f;
		ret.g = ret.g < 0.0f ? 0.0f : ret.g;
		ret.g = ret.g > 255.0f ? 255.0f : ret.g;
	} else {
		ret.g = temp - 60.0f;
		ret.g = 288.1221695283f * lm_powf(ret.g, -0.0755148492f);
		ret.g = ret.g < 0.0f ? 0.0f : ret.g;
		ret.g = ret.g > 255.0f ? 255.0f : ret.g;
	}
	if (temp >= 66.0f) {
		ret.b = 255.0f;
	} else {
		if (temp <= 19.0f) {
			ret.b = 0.0f;
		} else {
			ret.b = temp - 10.0f;
			ret.b = 138.5177312231f * lm_logf(ret.b) - 305.0447927307f;
			ret.b = ret.b < 0.0f ? 0.0f : ret.b;
			ret.b = ret.b > 255.0f ? 255.0f : ret.b;
		}
	}
	return (col){ ret.r / 255.0f, ret.g / 255.0f, ret.b / 255.0f, 0 };
}

/* ---- sampler: common.h:22-27, pcg_basic.c:42-68, random.c:16-21 ------------------------------------ */
struct rng { uint64_t state; struct cro_counters *ctr; }; /* inc is always 1 (initseq 0) */

static inline uint64_t hash64(uint64_t x) {
	x = (x ^ (x >> 30)) * UINT64_C(0xbf58476d1ce4e5b9);
	x = (x ^ (x >> 27)) * UINT64_C(0x94d049bb133111eb);
	x = x ^ (x >> 31);
	return x;
}
static inline uint32_t pcg32(struct rng *r) {
	uint64_t old = r->state;
	r->state = old * 6364136223846793005ULL + 1u;
	uint32_t xorshifted = (uint32_t)(((old >> 18u) ^ old) >> 27u);
	uint32_t rot = (uint32_t)(old >> 59u);
	return (xorshifted >> rot) | (xorshifted << ((-rot) & 31));
}
static inline void rng_init(struct rng *r, uint32_t pixIdx, int pass, int maxPasses) { /* sampler.c:41-44 */
	uint32_t seed32 = pixIdx * (uint32_t)maxPasses + (uint32_t)pass; /* 32-bit wrap is reference behaviour */
	uint64_t seed = hash64((uint64_t)seed32);
	r->state = 0u;
	pcg32(r);
	r->state += seed;
	pcg32(r);
}
static inline float draw(struct rng *r) {
	if (r->ctr) r->ctr->draws++;
	return (1.0f / (1ull << 32)) * pcg32(r); /* may equal 1.0f */
}

static inline v3 random_on_unit_sphere(struct rng *r) {                                       /* vector.h:243 */
	const float sx = draw(r);
	const float sy = draw(r);
	const float a = sx * (2.0f * PI);
	const float s = 2.0f * sqrtf(MAX_(0.0f, sy * (1.0f - sy)));
	return (v3){ lm_cosf(a) * s, lm_sinf(a) * s, 1.0f - 2.0f * sy };
}

/* ---- transforms.c:76-116 ----------------------------------------------------------------------------- */
static inline v3 xf_point(const float *m, v3 v) {
	return (v3){ (m[0] * v.x) + (m[1] * v.y) + (m[2] * v.z) + m[3],
				 (m[4] * v.x) + (m[5] * v.y) + (m[6] * v.z) + m[7],
				 (m[8] * v.x) + (m[9] * v.y) + (m[10] * v.z) + m[11] };
}
static inline v3 xf_vector(const float *m, v3 v) {
	return (v3){ (m[0] * v.x) + (m[1] * v.y) + (m[2] * v.z),
				 (m[4] * v.x) + (m[5] * v.y) + (m[6] * v.z),
				 (m[8] * v.x) + (m[9] * v.y) + (m[10] * v.z) };
}
static inline v3 xf_vector_transpose(const float *m, v3 v) {                                   /* :106-111 */
	return (v3){ (m[0] * v.x) + (m[4] * v.y) + (m[8] * v.z),
				 (m[1] * v.x) + (m[5] * v.y) + (m[9] * v.z),
				 (m[2] * v.x) + (m[6] * v.y) + (m[10] * v.z) };
}

/* ---- hit record (hitrecord.h:14-23, flattened) ------------------------------------------------------ */
struct ray { v3 o, d; };
struct hit {
	struct ray incident;
	int material;      /* global material index (the reference copies the 144-byte struct) */
	v3 p, n;
	v2 uv;
	v2 bary;           /* barycentric (u, v) of the winning triangle, before texmap_mesh replaces uv */
	float dist;
	int poly;          /* global poly index or -1 */
	int inst;
};

/* ---- camera.c:50-87 ------------------------------------------------------------------------------------ */
static inline float signf_(float v) { return (v >= 0.0f) ? 1.0f : -1.0f; }
static inline float triangle_distribution(float v) {
	const float orig = v * 2.0f - 1.0f;
	v = orig / sqrtf(fabsf(orig));
	v = clampf(v, -1.0f, 1.0f);
	v = v - signf_(orig);
	return v;
}
static struct ray camera_ray(const struct crs_camera *cam, int x, int y, struct rng *r) {
	struct ray ray = { { 0, 0, 0 }, { 0, 0, 0 } };
	const v3 right = { cam->right[0], cam->right[1], cam->right[2] };
	const v3 up = { cam->up[0], cam->up[1], cam->up[2] };
	const v3 forward = { cam->forward[0], cam->forward[1], cam->forward[2] };
	const float jitterX = triangle_distribution(draw(r));
	const float jitterY = triangle_distribution(draw(r));
	v3 pixX = v3scale(right, (cam->sensor_x / cam->width));
	v3 pixY = v3scale(up, (cam->sensor_y / cam->height));
	v3 pixV = v3add(forward, v3add(v3scale(pixX, x - cam->width * 0.5f + jitterX + 0.5f),
								   v3scale(pixY, y - cam->height * 0.5f + jitterY + 0.5f)));
	ray.d = v3norm(pixV);
	if (cam->aperture > 0.0f) {
		float ft = cam->focal_distance / v3dot(ray.d, forward);
		v3 focus = v3add(ray.o, v3scale(ray.d, ft));
		float rr = sqrtf(draw(r));                           /* randomCoordOnUnitDisc, vector.h:194-198 */
		float theta = ((draw(r)) * (2.0f * PI - 0.0f)) + 0.0f; /* rndFloatRange(0, 2π) */
		v2 lens = { (rr * lm_cosf(theta)) * cam->aperture, (rr * lm_sinf(theta)) * cam->aperture };
		ray.o = v3add(ray.o, v3add(v3scale(right, lens.x), v3scale(up, lens.y)));
		ray.d = v3norm(v3sub(focus, ray.o));
	}
	ray.o = xf_point(cam->A, ray.o);
	ray.d = xf_vector(cam->A, ray.d);
	return ray;
}

/* ---- poly.c:17-53 ------------------------------------------------------------------------------------------ */
static inline v3 vtx(const float *a, int i) { return (v3){ a[3 * (size_t)i], a[3 * (size_t)i + 1], a[3 * (size_t)i + 2] }; }

static bool ray_triangle(const struct crs_scene *s, const struct ray *ray, int polyIdx, struct hit *isect) {
	const struct crs_poly *p = &s->polys[polyIdx];
	v3 v0 = vtx(s->vertices, p->v[0]), v1 = vtx(s->vertices, p->v[1]), v2_ = vtx(s->vertices, p->v[2]);
	v3 e1 = v3sub(v0, v1);
	v3 e2 = v3sub(v2_, v0);
	v3 n = v3cross(e1, e2);
	v3 c = v3sub(v0, ray->o);
	v3 r = v3cross(ray->d, c);
	float invDet = 1.0f / v3dot(n, ray->d);
	float u = v3dot(r, e2) * invDet;
	float v = v3dot(r, e1) * invDet;
	float w = 1.0f - u - v;
	if (u >= 0.0f && v >= 0.0f && u + v <= 1.0f) {
		float t = v3dot(n, c) * invDet;
		if (t >= 0.0f && t < isect->dist) {
			isect->uv = (v2){ u, v };
			isect->dist = t;
			if (p->has_normals) {
				v3 up = v3scale(vtx(s->normals, p->n[1]), u);
				v3 vp = v3scale(vtx(s->normals, p->n[2]), v);
				v3 wp = v3scale(vtx(s->normals, p->n[0]), w);
				isect->n = v3add(v3add(up, vp), wp);
			} else {
				isect->n = n;
			}
			isect->p = v3add(ray->o, v3scale(ray->d, t));
			return true;
		}
	}
	return false;
}

/* ---- sphere.c:20-61 ------------------------------------------------------------------------------------------ */
static bool ray_sphere(const struct ray *ray, float radius, struct hit *isect) {
	float A = v3dot(ray->d, ray->d);
	float B = 2.0f * v3dot(ray->d, ray->o);
	float C = v3dot(ray->o, ray->o) - (radius * radius);
	float disc = B * B - 4.0f * A * C;
	if (disc < 0.0f) return false;
	float sq = sqrtf(disc);
	float t0 = (-B + sq) / 2.0f;
	float t1 = (-B - sq) / 2.0f;
	if (t0 > t1 && t1 > 0.0f) t0 = t1;
	if (t0 < 0.00001f || t0 > isect->dist) return false;
	isect->dist = t0;
	isect->p = v3add(ray->o, v3scale(ray->d, isect->dist));
	isect->n = v3norm(isect->p);
	isect->poly = -1;
	return true;
}

/* ---- bvh.c:318-441 -------------------------------------------------------------------------------------------- */
static inline bool node_test(const struct crs_bvh_node *node, v3 invDir, v3 scaledStart, const int *oct,
							 float maxDist, float *tEntry) {
	/* strict reference build: FP_FAST_FMAF undefined → plain a*b+c (bvh.c:318-324) */
	float tMinX = node->bounds[0 + oct[0]] * invDir.x + scaledStart.x;
	float tMaxX = node->bounds[0 + 1 - oct[0]] * invDir.x + scaledStart.x;
	float tMinY = node->bounds[2 + oct[1]] * invDir.y + scaledStart.y;
	float tMaxY = node->bounds[2 + 1 - oct[1]] * invDir.y + scaledStart.y;
	float tMinZ = node->bounds[4 + oct[2]] * invDir.z + scaledStart.z;
	float tMaxZ = node->bounds[4 + 1 - oct[2]] * invDir.z + scaledStart.z;
	float tMin = tMinX > tMinY ? tMinX : tMinY;
	float tMax = tMaxX < tMaxY ? tMaxX : tMaxY;
	tMin = tMin > tMinZ ? tMin : tMinZ;
	tMax = tMax < tMaxZ ? tMax : tMaxZ;
	tMin = tMin > 0 ? tMin : 0;
	tMax = tMax < maxDist ? tMax : maxDist;
	*tEntry = tMin;
	return tMin <= tMax;
}

/* optional event trace of the traversal, at the granularity of the GPU kernel's state machine (crgpu_trace.cuh): used by
 * tools/k2_warp_model.py to study warp scheduling policies offline.  Event bytes: 0 = top-level child-pair step,
 * 1 = mesh instance step, 2 = sphere instance step, 64+k = bottom-level child-pair step that tested k triangles (k <= 63). */
struct cro_trace { uint8_t *buf; size_t cap, len; size_t pair_at; uint16_t x, y, pass; };
/* dev = 1: the device traversal's slab test (cro_closest_hit semantics 1); 0 everywhere else */
struct trav_ctx { const struct crs_scene *s; struct cro_counters *ctr; struct cro_trace *tr; int dev; };

/* The slab test of the device traversal (cr_node_test, crgpu_trace.cuh), which deviates from node_test in exactly two ways
 * (DESIGN.md §2): every bound*invDir+scaledStart is ONE fused rounding (fmaf), and an axis whose scaledStart = -o/d is not
 * finite (1/d is +-inf, or o*(1/d) overflows) is culled exactly, inside the slab iff lo <= o <= hi, instead of through the
 * NaN-tolerant min/max chain. */
static inline bool node_test_dev(const struct crs_bvh_node *node, v3 o, v3 invDir, v3 scaledStart, const int *oct,
								 float maxDist, float *tEntry) {
	const float *b = node->bounds;
	float tMinX = fmaf(b[0 + oct[0]], invDir.x, scaledStart.x);
	float tMaxX = fmaf(b[0 + 1 - oct[0]], invDir.x, scaledStart.x);
	float tMinY = fmaf(b[2 + oct[1]], invDir.y, scaledStart.y);
	float tMaxY = fmaf(b[2 + 1 - oct[1]], invDir.y, scaledStart.y);
	float tMinZ = fmaf(b[4 + oct[2]], invDir.z, scaledStart.z);
	float tMaxZ = fmaf(b[4 + 1 - oct[2]], invDir.z, scaledStart.z);
	if (!isfinite(scaledStart.x)) { const bool in = b[0] <= o.x && o.x <= b[1]; tMinX = in ? -INFINITY : INFINITY; tMaxX = in ? INFINITY : -INFINITY; }
	if (!isfinite(scaledStart.y)) { const bool in = b[2] <= o.y && o.y <= b[3]; tMinY = in ? -INFINITY : INFINITY; tMaxY = in ? INFINITY : -INFINITY; }
	if (!isfinite(scaledStart.z)) { const bool in = b[4] <= o.z && o.z <= b[5]; tMinZ = in ? -INFINITY : INFINITY; tMaxZ = in ? INFINITY : -INFINITY; }
	float tMin = tMinX > tMinY ? tMinX : tMinY;
	float tMax = tMaxX < tMaxY ? tMaxX : tMaxY;
	tMin = tMin > tMinZ ? tMin : tMinZ;
	tMax = tMax < tMaxZ ? tMax : tMaxZ;
	tMin = tMin > 0 ? tMin : 0;
	tMax = tMax < maxDist ? tMax : maxDist;
	*tEntry = tMin;
	return tMin <= tMax;
}
#define NODE_TEST(c, nd, o, invDir, scaledStart, oct, maxDist, tEntry) \
	((c)->dev ? node_test_dev((nd), (o), (invDir), (scaledStart), (oct), (maxDist), (tEntry)) \
	          : node_test((nd), (invDir), (scaledStart), (oct), (maxDist), (tEntry)))
static inline void tr_event(const struct trav_ctx *c, uint8_t code) {
	if (c->tr && c->tr->len < c->tr->cap) { c->tr->pair_at = c->tr->len; c->tr->buf[c->tr->len++] = code; }
}
static inline void tr_tri(const struct trav_ctx *c, size_t at) {
	if (c->tr && at < c->tr->cap && c->tr->buf[at] < 127) c->tr->buf[at]++;
}

static bool leaf_bottom(const struct trav_ctx *c, const struct crs_mesh *mesh, const struct crs_bvh *bvh,
						const struct crs_bvh_node *leaf, const struct ray *ray, struct hit *isect) { /* bvh.c:443-462 */
	bool found = false;
	int count = (int)(leaf->prim_count_leaf & CRS_BVH_COUNT_MASK);
	for (int i = 0; i < count; ++i) {
		int local = c->s->prim_indices[bvh->prim_offset + leaf->first_child_or_prim + (uint32_t)i];
		int polyIdx = (int)mesh->poly_offset + local;
		if (c->ctr) c->ctr->tri_tests++;
		if (c->tr) tr_tri(c, c->tr->pair_at);
		if (ray_triangle(c->s, ray, polyIdx, isect)) {
			isect->poly = polyIdx;
			found = true;
		}
	}
	return found;
}

static bool traverse(const struct trav_ctx *c, uint32_t bvhIdx, int meshIdx /* -1: top level */,
					 const struct ray *ray, struct hit *isect);

static v2 texmap_sphere(v3 ud) {                                                              /* instance.c:33-43 */
	float phi = lm_atan2f(ud.z, ud.x);
	float theta = lm_asinf(ud.y);
	float v = (theta + PI / 2.0f) / PI;
	float u = 1.0f - (phi + PI) / (PI * 2.0f);
	u = wrapMinMax(u, 0.0f, 1.0f);
	v = wrapMinMax(v, 0.0f, 1.0f);
	return (v2){ u, v };
}

static bool intersect_sphere_inst(const struct trav_ctx *c, const struct crs_instance *inst,
								  const struct ray *ray, struct hit *isect) {                  /* instance.c:45-60 */
	const struct crs_sphere *sp = &c->s->spheres[inst->object];
	struct ray copy = { xf_point(inst->Ainv, ray->o), xf_vector(inst->Ainv, ray->d) };
	copy.o = v3add(copy.o, v3scale(copy.d, sp->ray_offset));
	if (c->ctr) c->ctr->sphere_tests++;
	tr_event(c, 2);
	if (ray_sphere(&copy, sp->radius, isect)) {
		isect->uv = texmap_sphere(isect->n);
		isect->poly = -1;
		isect->material = (int)sp->material;
		isect->p = xf_point(inst->A, isect->p);
		isect->n = xf_vector_transpose(inst->Ainv, isect->n);
		return true;
	}
	return false;
}

static v2 texmap_mesh(const struct crs_scene *s, const struct crs_mesh *mesh, const struct hit *isect) { /* instance.c:150-167 */
	if (mesh->texcoord_count == 0) return (v2){ -1.0f, -1.0f };
	const struct crs_poly *p = &s->polys[isect->poly];
	if (p->t[0] == -1) return (v2){ -1.0f, -1.0f };
	const float u = isect->uv.x;
	const float v = isect->uv.y;
	const float w = 1.0f - u - v;
	const float *tc = s->texcoords;
	v2 uc = { tc[2 * (size_t)p->t[1]] * u, tc[2 * (size_t)p->t[1] + 1] * u };
	v2 vc = { tc[2 * (size_t)p->t[2]] * v, tc[2 * (size_t)p->t[2] + 1] * v };
	v2 wc = { tc[2 * (size_t)p->t[0]] * w, tc[2 * (size_t)p->t[0] + 1] * w };
	return (v2){ (uc.x + vc.x) + wc.x, (uc.y + vc.y) + wc.y };
}

static bool intersect_mesh_inst(const struct trav_ctx *c, const struct crs_instance *inst,
								const struct ray *ray, struct hit *isect) {                    /* instance.c:169-185 */
	const struct crs_mesh *mesh = &c->s->meshes[inst->object];
	struct ray copy = { xf_point(inst->Ainv, ray->o), xf_vector(inst->Ainv, ray->d) };
	copy.o = v3add(copy.o, v3scale(copy.d, mesh->ray_offset));
	if (c->ctr) c->ctr->inst_visits++;
	tr_event(c, 1);
	if (traverse(c, mesh->bvh, (int)inst->object, &copy, isect)) {
		isect->bary = isect->uv;
		isect->uv = texmap_mesh(c->s, mesh, isect);
		isect->material = (int)(mesh->material_offset + c->s->polys[isect->poly].material);
		isect->p = xf_point(inst->A, isect->p);
		isect->n = xf_vector_transpose(inst->Ainv, isect->n);
		isect->n = v3norm(isect->n);
		return true;
	}
	return false;
}

static bool leaf_top(const struct trav_ctx *c, const struct crs_bvh *bvh, const struct crs_bvh_node *leaf,
					 const struct ray *ray, struct hit *isect) {                               /* bvh.c:468-486 */
	bool found = false;
	int count = (int)(leaf->prim_count_leaf & CRS_BVH_COUNT_MASK);
	for (int i = 0; i < count; ++i) {
		int cur = c->s->prim_indices[bvh->prim_offset + leaf->first_child_or_prim + (uint32_t)i];
		const struct crs_instance *inst = &c->s->instances[cur];
		bool h = inst->kind == CRS_INST_MESH ? intersect_mesh_inst(c, inst, ray, isect)
											 : intersect_sphere_inst(c, inst, ray, isect);
		if (h) {
			isect->inst = cur;
			found = true;
		}
	}
	return found;
}

#define MAX_BVH_DEPTH 64

static bool traverse(const struct trav_ctx *c, uint32_t bvhIdx, int meshIdx, const struct ray *ray, struct hit *isect) {
	const struct crs_bvh *bvh = &c->s->bvhs[bvhIdx];
	const struct crs_bvh_node *nodes = c->s->bvh_nodes + bvh->node_offset;
	const struct crs_mesh *mesh = meshIdx >= 0 ? &c->s->meshes[meshIdx] : NULL;
#define LEAF(nd) (mesh ? leaf_bottom(c, mesh, bvh, (nd), ray, isect) : leaf_top(c, bvh, (nd), ray, isect))
	if (bvh->node_count < 1) {                                                              /* bvh.c:362-365 */
		isect->inst = -1;
		return false;
	}
	const struct crs_bvh_node *stack[MAX_BVH_DEPTH + 1];
	int stackSize = 0;
	int oct[3] = { signbit(ray->d.x) ? 1 : 0, signbit(ray->d.y) ? 1 : 0, signbit(ray->d.z) ? 1 : 0 };
	v3 invDir = { 1.0f / ray->d.x, 1.0f / ray->d.y, 1.0f / ray->d.z };
	v3 scaledStart = v3scale(v3mul(ray->o, invDir), -1.0f);
	float maxDist = isect->dist;

	if (bvh->node_count == 1) {                                                             /* bvh.c:382-387 */
		float tEntry;
		if (mesh) tr_event(c, 64);                               /* single-leaf BVH: one step that tests the leaf's triangles */
		if (NODE_TEST(c, nodes, ray->o, invDir, scaledStart, oct, maxDist, &tEntry)) return LEAF(nodes);
		return false;
	}
	const struct crs_bvh_node *node = nodes;
	bool hasHit = false;
	while (true) {
		unsigned firstChild = node->first_child_or_prim;
		const struct crs_bvh_node *left = &nodes[firstChild];
		const struct crs_bvh_node *right = &nodes[firstChild + 1];
		if (c->ctr) c->ctr->node_pairs++;
		tr_event(c, mesh ? 64 : 0);
		float tL, tR;
		bool hitL = NODE_TEST(c, left, ray->o, invDir, scaledStart, oct, maxDist, &tL);
		bool hitR = NODE_TEST(c, right, ray->o, invDir, scaledStart, oct, maxDist, &tR);
		if (hitL) {
			if (left->prim_count_leaf & CRS_BVH_LEAF_BIT) {
				if (LEAF(left)) { maxDist = isect->dist; hasHit = true; }
				left = NULL;
			}
		} else left = NULL;
		if (hitR) {
			if (right->prim_count_leaf & CRS_BVH_LEAF_BIT) {
				if (LEAF(right)) { maxDist = isect->dist; hasHit = true; }
				right = NULL;
			}
		} else right = NULL;
		if ((right != NULL) & (left != NULL)) {
			if (tL > tR) { node = left; left = right; right = node; }
			node = left;
			stack[stackSize++] = right;
			if (c->ctr && (uint64_t)stackSize > c->ctr->max_stack) c->ctr->max_stack = (uint64_t)stackSize;
		} else if ((right != NULL) ^ (left != NULL)) {
			node = right != NULL ? right : left;
		} else {
			if (stackSize == 0) break;
			node = stack[--stackSize];
		}
	}
#undef LEAF
	return hasHit;
}

/* ---- texture.c:32-79 ---------------------------------------------------------------------------------------------- */
/* (size_t)float as GCC emits it on x86-64 (cvttss2si): negative values wrap modulo 2^64 */
static inline uint64_t f2sz(float x) {
	if (x < 9223372036854775808.0f) return (uint64_t)(int64_t)x;
	return ((uint64_t)(int64_t)(x - 9223372036854775808.0f)) ^ (UINT64_C(1) << 63);
}

static col texel(const struct crs_scene *s, const struct crs_texture *t, uint64_t x, uint64_t y) {
	col o = { 0, 0, 0, 0 };
	x = x % t->width;
	y = y % t->height;
	const uint8_t *base = s->texdata + t->data_offset;
	size_t idx = (size_t)((x + ((t->height - 1) - y) * t->width) * t->channels);
	if (t->channels == 1) {
		if (t->is_float) o.r = ((const float *)base)[idx];
		else o.r = base[idx] / 255.0f;
		o.g = o.r; o.b = o.r; o.a = 1.0f;
	} else if (t->is_float) {
		const float *f = (const float *)base;
		o.r = f[idx]; o.g = f[idx + 1]; o.b = f[idx + 2];
		o.a = t->has_alpha ? f[idx + 3] : 1.0f;
	} else {
		o.r = base[idx] / 255.0f; o.g = base[idx + 1] / 255.0f; o.b = base[idx + 2] / 255.0f;
		o.a = t->has_alpha ? base[idx + 3] / 255.0f : 1.0f;
	}
	return o;
}

static col texture_get(const struct crs_scene *s, const struct crs_texture *t, float x, float y, bool filtered) {
	if (!filtered) return texel(s, t, f2sz(x), f2sz(y));
	x = x * t->width;
	y = y * t->height;
	float xcopy = x - 0.5f;
	float ycopy = y - 0.5f;
	int xint = (int)xcopy;
	int yint = (int)ycopy;
	col tl = texel(s, t, (uint64_t)(int64_t)xint, (uint64_t)(int64_t)yint);
	col tr = texel(s, t, (uint64_t)(int64_t)(xint + 1), (uint64_t)(int64_t)yint);
	col bl = texel(s, t, (uint64_t)(int64_t)xint, (uint64_t)(int64_t)(yint + 1));
	col br = texel(s, t, (uint64_t)(int64_t)(xint + 1), (uint64_t)(int64_t)(yint + 1));
	return cmix(cmix(tl, tr, xcopy - xint), cmix(bl, br, xcopy - xint), ycopy - yint);
}

/* ---- nodes ------------------------------------------------------------------------------------------------------------ */
static float eval_value(const struct crs_scene *s, int node, const struct hit *rec);
static inline float schlick(float cosine, float IOR);

/* vector nodes (vectornode.c:38-42, input/normal.c:36-40, converter/vecmath.c:43-83): struct vectorValue's .v member; the ops that
 * produce the scalar .f (dot, length) leave .v zero-initialised, and no node of the reference reads .f */
static v3 eval_vector(const struct crs_scene *s, int node, const struct hit *rec) {
	const struct crs_node *n = &s->nodes[node];
	switch (n->kind) {
	case CRS_VECTOR_CONSTANT: return (v3){ n->f[0], n->f[1], n->f[2] };
	case CRS_VECTOR_NORMAL: return rec->n;
	case CRS_VECTOR_VECMATH: {
		const v3 a = eval_vector(s, n->in[0], rec);
		const v3 b = eval_vector(s, n->in[1], rec);
		switch (n->options) {
		case CRS_VEC_ADD: return v3add(a, b);
		case CRS_VEC_SUBTRACT: return v3sub(a, b);
		case CRS_VEC_MULTIPLY: return (v3){ a.x * b.x, a.y * b.y, a.z * b.z };
		case CRS_VEC_AVERAGE: return v3scale(v3add(a, b), 0.5f);
		case CRS_VEC_CROSS: return v3cross(a, b);
		case CRS_VEC_NORMALIZE: return v3norm(a);
		case CRS_VEC_REFLECT: return v3reflect(a, b);
		case CRS_VEC_ABS: return (v3){ fabsf(a.x), fabsf(a.y), fabsf(a.z) };
		default: return (v3){ 0, 0, 0 };                     /* VecDot, VecLength: .f only */
		}
	}
	default: return (v3){ 0, 0, 0 };
	}
}

static col eval_color(const struct crs_scene *s, int node, const struct hit *rec) {
	const struct crs_node *n = &s->nodes[node];
	switch (n->kind) {
	case CRS_COLOR_CONSTANT:                                                          /* constant.c:39-42 */
		return (col){ n->f[0], n->f[1], n->f[2], n->f[3] };
	case CRS_COLOR_IMAGE: {                                                           /* image.c:31-48 */
		if (n->tex < 0) return (col){ 1.0f, 0.0f, 0.5f, 1.0f };
		const struct crs_texture *t = &s->textures[n->tex];
		col out;
		if (n->options & CRS_IMG_NO_BILINEAR) {
			float x = rec->uv.x * t->width;
			float y = rec->uv.y * t->height;
			out = texture_get(s, t, x, y, false);
		} else {
			out = texture_get(s, t, rec->uv.x, rec->uv.y, true);
		}
		if (n->options & CRS_IMG_SRGB_TRANSFORM)
			out = (col){ srgb_to_linear(out.r), srgb_to_linear(out.g), srgb_to_linear(out.b), out.a };
		return out;
	}
	case CRS_COLOR_CHECKER: {                                                         /* checker.c:31-54 */
		const float coef = eval_value(s, n->in[2], rec);
		float sines;
		if (rec->uv.x >= 0) sines = lm_sinf(coef * rec->uv.x) * lm_sinf(coef * rec->uv.y);
		else sines = lm_sinf(coef * rec->p.x) * lm_sinf(coef * rec->p.y) * lm_sinf(coef * rec->p.z);
		return sines < 0.0f ? eval_color(s, n->in[0], rec) : eval_color(s, n->in[1], rec);
	}
	case CRS_COLOR_GRADIENT: {                                                        /* gradient.c:40-45 */
		v3 unit = v3norm(rec->incident.d);
		float t = 0.5f * (unit.y + 1.0f);
		col down = { n->f[0], n->f[1], n->f[2], n->f[3] }, up = { n->f[4], n->f[5], n->f[6], n->f[7] };
		return cadd(ccoef(1.0f - t, down), ccoef(t, up));
	}
	case CRS_COLOR_BLACKBODY:                                                         /* blackbody.c:38-42 */
		return color_for_kelvin(eval_value(s, n->in[0], rec));
	case CRS_COLOR_VECTOCOLOR: {                                                      /* vectocolor.c:38-43 */
		const v3 v = eval_vector(s, n->in[0], rec);
		return (col){ v.x, v.y, v.z, 0.0f };
	}
	case CRS_COLOR_COMBINE_VALUE: {                                                   /* combine.c:38-43 */
		const float v = eval_value(s, n->in[0], rec);
		return (col){ v, v, v, 1.0f };
	}
	case CRS_COLOR_COMBINE_RGB: {                                                     /* combinergb.c:44-53: R, G, B in this order */
		const float r = eval_value(s, n->in[0], rec);
		const float g = eval_value(s, n->in[1], rec);
		const float b = eval_value(s, n->in[2], rec);
		return (col){ r, g, b, 1.0f };
	}
	default:
		return (col){ 0, 0, 0, 1 };
	}
}

static float eval_value(const struct crs_scene *s, int node, const struct hit *rec) {
	const struct crs_node *n = &s->nodes[node];
	switch (n->kind) {
	case CRS_VALUE_CONSTANT: return n->f[0];
	case CRS_VALUE_GRAYSCALE: return to_grayscale(eval_color(s, n->in[0], rec)).r;     /* grayscale.c:40-43 */
	case CRS_VALUE_ALPHA: return eval_color(s, n->in[0], rec).a;                        /* alpha.c:38-41 */
	case CRS_VALUE_MATH: {                                                              /* math.c:44-97 */
		const float a = eval_value(s, n->in[0], rec);
		const float b = eval_value(s, n->in[1], rec);
		switch (n->options) {
		case CRS_MATH_ADD: return a + b;
		case CRS_MATH_SUBTRACT: return a - b;
		case CRS_MATH_MULTIPLY: return a * b;
		case CRS_MATH_DIVIDE: return a / b;
		case CRS_MATH_POWER: return lm_powf(a, b);
		case CRS_MATH_LOG: return lm_log10f(a);
		case CRS_MATH_SQRT: return sqrtf(a);
		case CRS_MATH_ABS: return fabsf(a);
		case CRS_MATH_MIN: return MIN_(a, b);
		case CRS_MATH_MAX: return MAX_(a, b);
		case CRS_MATH_SINE: return lm_sinf(a);
		case CRS_MATH_COSINE: return lm_cosf(a);
		case CRS_MATH_TANGENT: return lm_tanf(a);
		case CRS_MATH_TO_RADIANS: return (a * PI) / 180.0f;                             /* transforms.c:18-20 */
		case CRS_MATH_TO_DEGREES: return a * (180.0f / PI);                             /* transforms.c:22-24 */
		default: return 0.0f;
		}
	}
	case CRS_VALUE_FRESNEL: {                                                           /* fresnel.c:43-55: IOR is evaluated twice */
		const float IOR = eval_value(s, n->in[0], rec);
		float cosine;
		const float dn = v3dot(rec->incident.d, rec->n);
		if (dn > 0.0f) cosine = IOR * v3dot(rec->incident.d, rec->n) / v3len(rec->incident.d);
		else cosine = -(v3dot(rec->incident.d, rec->n) / v3len(rec->incident.d));
		return schlick(cosine, eval_value(s, n->in[0], rec));
	}
	case CRS_VALUE_RAYLENGTH: return rec->dist;                                         /* raylength.c:36-40 */
	default: return 0.0f;
	}
}

struct bsdf_sample { v3 out; col color; };

static bool refract_(v3 in, v3 normal, float niOverNt, v3 *refracted) {                 /* vector.h:252-266 */
	const v3 uv = v3norm(in);
	const float dt = v3dot(uv, normal);
	const float disc = 1.0f - niOverNt * niOverNt * (1.0f - dt * dt);
	if (disc > 0.0f) {
		const v3 A = v3scale(normal, dt);
		const v3 B = v3sub(uv, A);
		const v3 C = v3scale(B, niOverNt);
		const v3 D = v3scale(normal, sqrtf(disc));
		*refracted = v3sub(C, D);
		return true;
	}
	return false;
}
static inline float schlick(float cosine, float IOR) {                                  /* vector.h:268-272 */
	float r0 = (1.0f - IOR) / (1.0f + IOR);
	r0 = r0 * r0;
	return r0 + (1.0f - r0) * lm_pow5f((1.0f - cosine));
}

static struct bsdf_sample sample_bsdf(const struct crs_scene *s, int node, struct rng *r, struct hit *rec) {
	const struct crs_node *n = &s->nodes[node];
	switch (n->kind) {
	case CRS_BSDF_DIFFUSE: {                                                          /* diffuse.c:40-47 */
		const v3 dir = v3norm(v3add(rec->n, random_on_unit_sphere(r)));
		return (struct bsdf_sample){ dir, eval_color(s, n->in[0], rec) };
	}
	case CRS_BSDF_ISOTROPIC: {                                                        /* isotropic.c:40-47 */
		const v3 dir = v3norm(random_on_unit_sphere(r));
		return (struct bsdf_sample){ dir, eval_color(s, n->in[0], rec) };
	}
	case CRS_BSDF_EMISSIVE: {                                                         /* emission.c:42-49 */
		const v3 dir = v3norm(v3add(rec->n, random_on_unit_sphere(r)));
		float strength = eval_value(s, n->in[1], rec);
		return (struct bsdf_sample){ dir, ccoef(strength, eval_color(s, n->in[0], rec)) };
	}
	case CRS_BSDF_METAL: {                                                            /* metal.c:40-55 */
		const v3 nd = v3norm(rec->incident.d);
		v3 reflected = v3reflect(nd, rec->n);
		float rough = eval_value(s, n->in[1], rec);
		if (rough > 0.0f) reflected = v3add(reflected, v3scale(random_on_unit_sphere(r), rough));
		return (struct bsdf_sample){ reflected, eval_color(s, n->in[0], rec) };
	}
	case CRS_BSDF_GLASS: {                                                            /* glass.c:41-87 */
		/* glass.c:47 declares `refracted` uninitialised and reads it (:76-80) when refract() failed (total internal reflection)
		 * and the draw is exactly 1.0f (129 of 2^32 draws): the compiled reference then scatters along (0, 0, <stale stack word>),
		 * which is not a function of the path.  DEFINED here (DESIGN.md deviation #3, identical in crgpu_shade.cuh): total
		 * internal reflection always reflects, i.e. `refracted` starts out as `reflected`. */
		v3 outward;
		v3 reflected = v3reflect(rec->incident.d, rec->n);
		v3 refracted = reflected;
		float niOverNt, prob, cosine;
		float IOR = eval_value(s, n->in[2], rec);
		if (v3dot(rec->incident.d, rec->n) > 0.0f) {
			outward = v3neg(rec->n);
			niOverNt = IOR;
			cosine = IOR * v3dot(rec->incident.d, rec->n) / v3len(rec->incident.d);
		} else {
			outward = rec->n;
			niOverNt = 1.0f / IOR;
			cosine = -(v3dot(rec->incident.d, rec->n) / v3len(rec->incident.d));
		}
		if (refract_(rec->incident.d, outward, niOverNt, &refracted)) prob = schlick(cosine, IOR);
		else prob = 1.0f;
		float rough = eval_value(s, n->in[1], rec);
		if (rough > 0.0f) {
			v3 fuzz = v3scale(random_on_unit_sphere(r), rough);
			reflected = v3add(reflected, fuzz);
			refracted = v3add(refracted, fuzz);
		}
		v3 dir = draw(r) < prob ? reflected : refracted;
		return (struct bsdf_sample){ dir, eval_color(s, n->in[0], rec) };
	}
	case CRS_BSDF_PLASTIC: {                                                          /* plastic.c:42-87 */
		v3 outward, refracted;
		float niOverNt, prob, cosine;
		const float IOR = s->materials[rec->material].IOR;
		if (v3dot(rec->incident.d, rec->n) > 0.0f) {
			outward = v3neg(rec->n);
			niOverNt = IOR;
			cosine = IOR * v3dot(rec->incident.d, rec->n) / v3len(rec->incident.d);
		} else {
			outward = rec->n;
			niOverNt = 1.0f / IOR;
			cosine = -(v3dot(rec->incident.d, rec->n) / v3len(rec->incident.d));
		}
		if (refract_(rec->incident.d, outward, niOverNt, &refracted)) prob = schlick(cosine, IOR);
		else prob = 1.0f;
		if (draw(r) < prob) {                                                         /* sampleShiny :42-56 */
			v3 reflected = v3reflect(rec->incident.d, rec->n);
			float rough = eval_color(s, n->in[1], rec).r;
			if (rough > 0.0f) reflected = v3add(reflected, v3scale(random_on_unit_sphere(r), rough));
			return (struct bsdf_sample){ reflected, (col){ 1.0f, 1.0f, 1.0f, 1.0f } };
		}
		return sample_bsdf(s, n->in[2], r, rec);
	}
	case CRS_BSDF_MIX: {                                                              /* mix.c:42-50 */
		const float lerp = eval_value(s, n->in[2], rec);
		if (draw(r) > lerp) return sample_bsdf(s, n->in[0], r, rec);
		return sample_bsdf(s, n->in[1], r, rec);
	}
	case CRS_BSDF_ADD: {                                                              /* add.c:42-49 */
		struct bsdf_sample A = sample_bsdf(s, n->in[0], r, rec);
		struct bsdf_sample B = sample_bsdf(s, n->in[1], r, rec);
		return (struct bsdf_sample){ v3add(A.out, B.out), cadd(A.color, B.color) };
	}
	case CRS_BSDF_TRANSPARENT:                                                        /* transparent.c:40-44 */
		return (struct bsdf_sample){ rec->incident.d, eval_color(s, n->in[0], rec) };
	case CRS_BSDF_BACKGROUND: {                                                       /* background.c:39-66 */
		v3 ud = v3norm(rec->incident.d);
		float rr = 1.0f;
		float phi = (lm_atan2f(ud.z, ud.x) / 4.0f) + eval_value(s, n->in[2], rec);
		float theta = lm_acosf((-ud.y / rr));
		float u = theta / PI;
		float v = (phi / (PI / 2.0f));
		u = wrapMinMax(u, 0.0f, 1.0f);
		v = wrapMinMax(v, 0.0f, 1.0f);
		rec->uv = (v2){ v, u };
		float strength = eval_value(s, n->in[1], rec);
		return (struct bsdf_sample){ (v3){ 0, 0, 0 }, ccoef(strength, eval_color(s, n->in[0], rec)) };
	}
	default:
		return (struct bsdf_sample){ (v3){ 0, 0, 0 }, (col){ 0, 0, 0, 1 } };
	}
}

/* ---- pathtrace.c:26-60 ---------------------------------------------------------------------------------------------------- */
static struct hit closest_isect(const struct trav_ctx *c, const struct ray *ray) {
	struct hit isect;
	memset(&isect, 0, sizeof isect);
	isect.incident = *ray;
	isect.inst = -1;
	isect.dist = FLT_MAX;
	isect.poly = -1;
	if (c->ctr) c->ctr->rays++;
	const uint64_t before = c->ctr ? c->ctr->node_pairs : 0;
	traverse(c, c->s->top_bvh, -1, ray, &isect);
	if (c->ctr && c->ctr->node_pairs - before > c->ctr->max_pairs_ray) c->ctr->max_pairs_ray = c->ctr->node_pairs - before;
	return isect;
}

/* One pass through pathTrace's loop body (pathtrace.c:37-57) at `depth`: returns false where the loop breaks.  `final` is only
 * read once `*has_final` is set (it is treated as (0, 0, 0, 1), pathtrace.c:34, before), which is how a path state that has not
 * received any radiance yet is handed between calls (cro_path_step); path_trace starts with it set.  `hit_out` (may be NULL)
 * receives the closest-hit record of the step's ray. */
static bool path_step(const struct trav_ctx *c, struct ray *ray, col *weight, col *final, int *has_final, int depth,
					  struct rng *r, struct cro_ray_record *hit_out) {
	const struct crs_scene *s = c->s;
	size_t hdr = 0;
	const size_t HDR = 36;
	int have_hdr = 0;
	if (c->tr && c->tr->len + HDR <= c->tr->cap) {           /* record header: x, y, pass, depth (u16), event count (u32), o, d (6 x f32) */
		hdr = c->tr->len;
		have_hdr = 1;
		const uint16_t h[4] = { c->tr->x, c->tr->y, c->tr->pass, (uint16_t)depth };
		const float od[6] = { ray->o.x, ray->o.y, ray->o.z, ray->d.x, ray->d.y, ray->d.z };
		memcpy(c->tr->buf + hdr, h, 8);
		memcpy(c->tr->buf + hdr + 12, od, 24);
		c->tr->len += HDR;
	}
	struct hit isect = closest_isect(c, ray);
	if (have_hdr) { const uint32_t n = (uint32_t)(c->tr->len - hdr - HDR); memcpy(c->tr->buf + hdr + 8, &n, 4); }
	if (c->ctr && (uint64_t)(depth + 1) > c->ctr->max_depth) c->ctr->max_depth = (uint64_t)(depth + 1);
	if (hit_out) {
		hit_out->t = isect.dist; hit_out->u = isect.bary.x; hit_out->v = isect.bary.y;
		hit_out->inst = isect.inst; hit_out->poly = -1; hit_out->material = -1;
		if (isect.inst >= 0) {
			hit_out->poly = s->instances[isect.inst].kind == CRS_INST_MESH ? isect.poly : -1;
			hit_out->material = isect.material;
		}
	}
	if (!*has_final) *final = (col){ 0, 0, 0, 1 };
	if (isect.inst < 0) {
		*final = cadd(*final, cmul(*weight, sample_bsdf(s, s->background, r, &isect).color));
		*has_final = 1;
		return false;
	}
	const struct crs_material *m = &s->materials[isect.material];
	/* The device adds emission only where it can change `final` (cr_shade_one: DevMaterial flag 2, or a weight that is not finite):
	 * x + w*0 == x for finite w and every x but -0, which a sum that starts at +0 never is.  `*has_final` follows that rule in
	 * both semantics, so a state without radiance always holds +0 (DESIGN.md §2, deviation 4); semantics 1 also skips the add. */
	const col e = { m->emission[0], m->emission[1], m->emission[2], m->emission[3] };
	const bool adds = !(e.r == 0.0f && e.g == 0.0f && e.b == 0.0f) || !(isfinite(weight->r) && isfinite(weight->g) && isfinite(weight->b));
	if (adds) *has_final = 1;
	if (adds || !c->dev) *final = cadd(*final, cmul(*weight, e));
	const struct bsdf_sample smp = sample_bsdf(s, m->bsdf, r, &isect);
	*ray = (struct ray){ isect.p, smp.out };
	const col att = smp.color;
	float probability = 1.0f;
	if (depth >= 4) {
		probability = MAX_(att.r, MAX_(att.g, att.b));
		if (draw(r) > probability) return false;
	}
	*weight = ccoef(1.0f / probability, cmul(att, *weight));
	return true;
}

static col path_trace(const struct trav_ctx *c, struct ray ray, int maxDepth, struct rng *r) {
	col weight = { 1, 1, 1, 1 };
	col final = { 0, 0, 0, 1 };
	int has_final = 1;
	for (int depth = 0; depth < maxDepth; ++depth)
		if (!path_step(c, &ray, &weight, &final, &has_final, depth, r, NULL)) break;
	return final;
}

/* ---- renderer.c:271-320 ------------------------------------------------------------------------------------------------------ */
struct job {
	const struct crs_scene *s;
	int x0, x1, ybegin, yend, pass_begin, pass_count;
	float *rgb;
	struct cro_counters ctr;
	bool count;
	int sem;                 /* libm and slab-test semantics (cro_render_sem) */
	uint32_t *flagged;       /* per framebuffer pixel: samples with a near-tie libm evaluation, or NULL */
};

static void *render_rows(void *arg) {
	struct job *j = arg;
	const struct crs_scene *s = j->s;
	struct trav_ctx c = { s, j->count ? &j->ctr : NULL, NULL, j->sem };
	lm_sem = j->sem;
	const int W = (int)s->prefs.image_width, H = (int)s->prefs.image_height;
	const int maxPasses = (int)s->prefs.sample_count, bounces = (int)s->prefs.bounces;
	for (int y = j->yend - 1; y > j->ybegin - 1; --y) {
		for (int x = j->x0; x < j->x1; ++x) {
			uint32_t pixIdx = (uint32_t)(y * W + x);
			float *px = j->rgb + ((size_t)x + (size_t)(H - (y + 1)) * (size_t)W) * 3;
			for (int pass = j->pass_begin; pass < j->pass_begin + j->pass_count; ++pass) {
				struct rng r = { 0, c.ctr };
				rng_init(&r, pixIdx, pass, maxPasses);
				col out = { px[0], px[1], px[2], 1.0f };
				lm_tie = 0;
				struct ray ray = camera_ray(&s->camera, x, y, &r);
				if (c.ctr) c.ctr->paths++;
				col smp = path_trace(&c, ray, bounces, &r);
				if (lm_tie && j->flagged) j->flagged[(size_t)x + (size_t)(H - (y + 1)) * (size_t)W]++;
				const int completed = pass + 1;
				out = ccoef((float)(completed - 1), out);
				out = cadd(out, smp);
				float t = 1.0f / completed;
				out = ccoef(t, out);
				px[0] = out.r; px[1] = out.g; px[2] = out.b;
			}
		}
	}
	return NULL;
}

struct runner { struct job *jobs; int first, step, n; };

static void *run_chunks(void *arg) {
	struct runner *r = arg;
	for (int i = r->first; i < r->n; i += r->step) render_rows(&r->jobs[i]);
	return NULL;
}

/* Traversal event trace of every ray of a region (single thread; pixels row-major y up, passes innermost), see struct cro_trace.
 * Returns the number of bytes written (records are dropped, not truncated, once the buffer is full). */
size_t cro_trace_region(const struct crs_scene *s, int x0, int y0, int x1, int y1, int pass_begin, int pass_count, uint8_t *buf, size_t cap) {
	struct cro_trace tr = { buf, cap, 0, 0, 0, 0, 0 };
	struct trav_ctx c = { s, NULL, &tr, 0 };
	const int W = (int)s->prefs.image_width;
	const int maxPasses = (int)s->prefs.sample_count, bounces = (int)s->prefs.bounces;
	for (int y = y0; y < y1; ++y)
		for (int x = x0; x < x1; ++x)
			for (int pass = pass_begin; pass < pass_begin + pass_count; ++pass) {
				struct rng r = { 0, NULL };
				rng_init(&r, (uint32_t)(y * W + x), pass, maxPasses);
				tr.x = (uint16_t)x; tr.y = (uint16_t)y; tr.pass = (uint16_t)pass;
				struct ray ray = camera_ray(&s->camera, x, y, &r);
				if (tr.len + 4096 > tr.cap) return tr.len;
				path_trace(&c, ray, bounces, &r);
			}
	return tr.len;
}

int cro_render(const struct crs_scene *s, int x0, int y0, int x1, int y1, int pass_begin, int pass_count,
			   float *rgb, int threads, struct cro_counters *counters) {
	return cro_render_sem(s, x0, y0, x1, y1, pass_begin, pass_count, rgb, threads, 0, NULL, counters);
}

int cro_render_sem(const struct crs_scene *s, int x0, int y0, int x1, int y1, int pass_begin, int pass_count,
				   float *rgb, int threads, int semantics, uint32_t *flagged, struct cro_counters *counters) {
	if (semantics != 0 && semantics != 1) return -1;
	if (threads < 1) threads = 1;
	int rows = y1 - y0;
	if (rows < 1 || x1 <= x0) return 0;
	if (threads > rows) threads = rows;
	/* interleaved row chunks so that threads finish together */
	int chunks = threads * 8;
	if (chunks > rows) chunks = rows;
	struct job *jobs = calloc((size_t)chunks, sizeof *jobs);
	for (int i = 0; i < chunks; ++i) {
		jobs[i] = (struct job){ .s = s, .x0 = x0, .x1 = x1, .ybegin = y0 + (int)((int64_t)rows * i / chunks),
			.yend = y0 + (int)((int64_t)rows * (i + 1) / chunks), .pass_begin = pass_begin, .pass_count = pass_count,
			.rgb = rgb, .count = counters != NULL, .sem = semantics, .flagged = flagged };
	}
	/* simple static round-robin over threads: each thread runs chunks t, t+threads, ... */
	pthread_t *tids = calloc((size_t)threads, sizeof *tids);
	struct runner *rs = calloc((size_t)threads, sizeof *rs);
	for (int t = 0; t < threads; ++t) {
		rs[t] = (struct runner){ jobs, t, threads, chunks };
		pthread_create(&tids[t], NULL, run_chunks, &rs[t]);
	}
	for (int t = 0; t < threads; ++t) pthread_join(tids[t], NULL);
	if (counters) {
		memset(counters, 0, sizeof *counters);
		for (int i = 0; i < chunks; ++i) {
			const struct cro_counters *k = &jobs[i].ctr;
			counters->paths += k->paths; counters->rays += k->rays; counters->node_pairs += k->node_pairs;
			counters->tri_tests += k->tri_tests; counters->sphere_tests += k->sphere_tests;
			counters->inst_visits += k->inst_visits; counters->draws += k->draws;
			if (k->max_depth > counters->max_depth) counters->max_depth = k->max_depth;
			if (k->max_stack > counters->max_stack) counters->max_stack = k->max_stack;
			if (k->max_pairs_ray > counters->max_pairs_ray) counters->max_pairs_ray = k->max_pairs_ray;
		}
	}
	free(rs); free(tids); free(jobs);
	return 0;
}

/* ---- known-answer helpers ------------------------------------------------------------------------------------------------------ */
void cro_sampler_kat(uint32_t pixIdx, int pass, int maxPasses, int n, float *out) {
	struct rng r = { 0, NULL };
	rng_init(&r, pixIdx, pass, maxPasses);
	for (int i = 0; i < n; ++i) out[i] = draw(&r);
}

void cro_trace_kat(const struct crs_scene *s, int x, int y, int pass, struct cro_hit_kat *k) {
	memset(k, 0, sizeof *k);
	const int W = (int)s->prefs.image_width;
	struct trav_ctx c = { s, NULL, NULL, 0 };
	k->x = x; k->y = y; k->pixIdx = y * W + x;
	struct rng r = { 0, NULL };
	rng_init(&r, (uint32_t)k->pixIdx, pass, (int)s->prefs.sample_count);
	struct ray ray = camera_ray(&s->camera, x, y, &r);
	k->o[0] = ray.o.x; k->o[1] = ray.o.y; k->o[2] = ray.o.z;
	k->d[0] = ray.d.x; k->d[1] = ray.d.y; k->d[2] = ray.d.z;
	struct hit isect = closest_isect(&c, &ray);
	k->instIndex = isect.inst;
	struct bsdf_sample smp;
	if (isect.inst < 0) {
		k->polyIndex = -1;
		smp = sample_bsdf(s, s->background, &r, &isect);
	} else {
		k->polyIndex = isect.poly;
		k->distance = isect.dist; k->uv[0] = isect.uv.x; k->uv[1] = isect.uv.y;
		k->hitPoint[0] = isect.p.x; k->hitPoint[1] = isect.p.y; k->hitPoint[2] = isect.p.z;
		k->normal[0] = isect.n.x; k->normal[1] = isect.n.y; k->normal[2] = isect.n.z;
		const struct crs_material *m = &s->materials[isect.material];
		k->emission[0] = m->emission[0]; k->emission[1] = m->emission[1]; k->emission[2] = m->emission[2];
		smp = sample_bsdf(s, m->bsdf, &r, &isect);
	}
	k->out[0] = smp.out.x; k->out[1] = smp.out.y; k->out[2] = smp.out.z;
	k->color[0] = smp.color.r; k->color[1] = smp.color.g; k->color[2] = smp.color.b; k->color[3] = smp.color.a;
	k->nextDraw = draw(&r);
}

/* ---- per-ray closest hit (getClosestIsect, pathtrace.c:26-30) over a batch of rays ------------------------------------------------ */
struct ray_job { const struct crs_scene *s; const float *rays; struct cro_ray_record *out; size_t lo, hi; int dev; struct cro_counters ctr; bool count; };

static void *closest_hit_rows(void *arg) {
	struct ray_job *j = arg;
	struct trav_ctx c = { j->s, j->count ? &j->ctr : NULL, NULL, j->dev };
	lm_sem = j->dev;
	for (size_t i = j->lo; i < j->hi; ++i) {
		const float *r = j->rays + 6 * i;
		const struct ray ray = { { r[0], r[1], r[2] }, { r[3], r[4], r[5] } };
		const struct hit h = closest_isect(&c, &ray);
		struct cro_ray_record *o = &j->out[i];
		o->t = h.dist;
		o->u = h.bary.x; o->v = h.bary.y;
		o->inst = h.inst;
		o->poly = -1; o->material = -1;
		if (h.inst >= 0) {
			o->poly = j->s->instances[h.inst].kind == CRS_INST_MESH ? h.poly : -1;
			o->material = h.material;
		}
	}
	return NULL;
}

int cro_closest_hit(const struct crs_scene *s, size_t n, const float *rays, int semantics, int threads,
					struct cro_ray_record *out, struct cro_counters *counters) {
	if (semantics != 0 && semantics != 1) return -1;
	if (counters) memset(counters, 0, sizeof *counters);
	if (n == 0) return 0;
	if (threads < 1) threads = 1;
	if ((size_t)threads > n) threads = (int)n;
	struct ray_job *jobs = calloc((size_t)threads, sizeof *jobs);
	pthread_t *tids = calloc((size_t)threads, sizeof *tids);
	if (!jobs || !tids) { free(jobs); free(tids); return -1; }
	for (int t = 0; t < threads; ++t) {
		jobs[t] = (struct ray_job){ .s = s, .rays = rays, .out = out, .lo = n * (size_t)t / (size_t)threads,
			.hi = n * (size_t)(t + 1) / (size_t)threads, .dev = semantics, .count = counters != NULL };
		pthread_create(&tids[t], NULL, closest_hit_rows, &jobs[t]);
	}
	for (int t = 0; t < threads; ++t) pthread_join(tids[t], NULL);
	if (counters) {
		for (int t = 0; t < threads; ++t) {
			const struct cro_counters *k = &jobs[t].ctr;
			counters->rays += k->rays; counters->node_pairs += k->node_pairs; counters->tri_tests += k->tri_tests;
			counters->sphere_tests += k->sphere_tests; counters->inst_visits += k->inst_visits;
			if (k->max_stack > counters->max_stack) counters->max_stack = k->max_stack;
			if (k->max_pairs_ray > counters->max_pairs_ray) counters->max_pairs_ray = k->max_pairs_ray;
		}
	}
	free(tids); free(jobs);
	return 0;
}

void cro_to_srgb8(const float *rgb, uint8_t *out, size_t pixels) {
	for (size_t i = 0; i < pixels * 3; ++i) {
		float c = linear_to_srgb(rgb[i]);
		out[i] = (unsigned char)MIN_(c * 255.0f, 255.0f);
	}
}

/* ---- path states: pathTrace's loop body one step at a time (the device's per-bounce kernels) ------------------------------------ */
static inline struct rng rng_of(uint64_t state) { struct rng r = { state, NULL }; return r; }

void cro_camera_states(const struct crs_scene *s, int x0, int y0, int x1, int y1, int pass_begin, int pass_count, int semantics,
					   struct cro_path_state *out) {
	const int W = (int)s->prefs.image_width;
	const int maxPasses = (int)s->prefs.sample_count;
	size_t k = 0;
	lm_sem = semantics;
	for (int y = y0; y < y1; ++y)
		for (int x = x0; x < x1; ++x)
			for (int pass = pass_begin; pass < pass_begin + pass_count; ++pass, ++k) {
				struct rng r = { 0, NULL };
				rng_init(&r, (uint32_t)(y * W + x), pass, maxPasses);
				lm_tie = 0;
				const struct ray ray = camera_ray(&s->camera, x, y, &r);
				struct cro_path_state *p = &out[k];
				memset(p, 0, sizeof *p);
				p->pad = (uint32_t)lm_tie;
				p->o[0] = ray.o.x; p->o[1] = ray.o.y; p->o[2] = ray.o.z;
				p->d[0] = ray.d.x; p->d[1] = ray.d.y; p->d[2] = ray.d.z;
				p->weight[0] = p->weight[1] = p->weight[2] = 1.0f;
				p->rng = r.state;
			}
	lm_sem = 0;
}

struct step_job {
	const struct crs_scene *s;
	const struct cro_path_state *in;
	struct cro_step_result *out;
	size_t lo, hi;
	int depth, maxDepth, bounces, sem;
};

static void *step_rows(void *arg) {
	struct step_job *j = arg;
	struct trav_ctx c = { j->s, NULL, NULL, j->sem };
	lm_sem = j->sem;
	for (size_t i = j->lo; i < j->hi; ++i) {
		const struct cro_path_state *p = &j->in[i];
		struct cro_step_result *o = &j->out[i];
		memset(o, 0, sizeof *o);
		struct ray ray = { { p->o[0], p->o[1], p->o[2] }, { p->d[0], p->d[1], p->d[2] } };
		col weight = { p->weight[0], p->weight[1], p->weight[2], 1.0f };
		col final = { p->L[0], p->L[1], p->L[2], 1.0f };
		int has = p->has_l ? 1 : 0;
		struct rng r = rng_of(p->rng);
		lm_tie = 0;
		bool alive = true;
		o->rec.inst = -1; o->rec.poly = -1; o->rec.material = -1;
		for (int depth = j->depth, k = 0; k < j->bounces; ++depth, ++k) {
			if (depth >= j->maxDepth) { alive = false; break; }
			alive = path_step(&c, &ray, &weight, &final, &has, depth, &r, k == 0 ? &o->rec : NULL)
					&& depth + 1 < j->maxDepth;
			if (!alive) break;
		}
		if (!alive && !has) final = (col){ 0, 0, 0, 1 };
		o->alive = alive;
		o->flag = (uint32_t)lm_tie;
		o->next.o[0] = ray.o.x; o->next.o[1] = ray.o.y; o->next.o[2] = ray.o.z;
		o->next.d[0] = ray.d.x; o->next.d[1] = ray.d.y; o->next.d[2] = ray.d.z;
		o->next.weight[0] = weight.r; o->next.weight[1] = weight.g; o->next.weight[2] = weight.b;
		o->next.has_l = (uint32_t)has;
		o->next.rng = r.state;
		o->next.L[0] = has ? final.r : p->L[0]; o->next.L[1] = has ? final.g : p->L[1]; o->next.L[2] = has ? final.b : p->L[2];
		if (!alive) { o->next.L[0] = final.r; o->next.L[1] = final.g; o->next.L[2] = final.b; }
	}
	return NULL;
}

int cro_path_step(const struct crs_scene *s, size_t n, const struct cro_path_state *states, int depth, int maxDepth, int bounces,
				  int semantics, int threads, struct cro_step_result *out) {
	if ((semantics != 0 && semantics != 1) || depth < 0 || bounces < 1) return -1;
	if (n == 0) return 0;
	if (threads < 1) threads = 1;
	if ((size_t)threads > n) threads = (int)n;
	struct step_job *jobs = calloc((size_t)threads, sizeof *jobs);
	pthread_t *tids = calloc((size_t)threads, sizeof *tids);
	if (!jobs || !tids) { free(jobs); free(tids); return -1; }
	for (int t = 0; t < threads; ++t) {
		jobs[t] = (struct step_job){ .s = s, .in = states, .out = out, .lo = n * (size_t)t / (size_t)threads,
			.hi = n * (size_t)(t + 1) / (size_t)threads, .depth = depth, .maxDepth = maxDepth, .bounces = bounces, .sem = semantics };
		pthread_create(&tids[t], NULL, step_rows, &jobs[t]);
	}
	for (int t = 0; t < threads; ++t) pthread_join(tids[t], NULL);
	free(tids); free(jobs);
	return 0;
}

/* ---- the libm stand-ins one by one (test sweeps) ------------------------------------------------------------------------------- */
int cro_libm(int fn, int semantics, size_t n, const float *x, const float *y, float *out, uint8_t *flag) {
	if ((semantics != 0 && semantics != 1) || fn < 0 || fn >= CRO_LIBM_COUNT) return -1;
	lm_sem = semantics;
	for (size_t i = 0; i < n; ++i) {
		lm_tie = 0;
		float r;
		switch (fn) {
		case CRO_LIBM_SIN: r = lm_sinf(x[i]); break;
		case CRO_LIBM_COS: r = lm_cosf(x[i]); break;
		case CRO_LIBM_TAN: r = lm_tanf(x[i]); break;
		case CRO_LIBM_LOG: r = lm_logf(x[i]); break;
		case CRO_LIBM_LOG10: r = lm_log10f(x[i]); break;
		case CRO_LIBM_ATAN2: r = lm_atan2f(x[i], y[i]); break;
		case CRO_LIBM_ACOS: r = lm_acosf(x[i]); break;
		case CRO_LIBM_ASIN: r = lm_asinf(x[i]); break;
		case CRO_LIBM_POW: r = lm_powf(x[i], y[i]); break;
		default: r = lm_pow5f(x[i]); break;
		}
		out[i] = r;
		if (flag) flag[i] = (uint8_t)lm_tie;
	}
	lm_sem = 0;
	return 0;
}
