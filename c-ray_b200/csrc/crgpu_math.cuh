/*
 * crgpu_math.cuh — device restatement of c-ray's inline fp32 math (reference src/datatypes/vector.h,
 * color.h, transforms.c) with IEEE semantics pinned so results match the -ffp-contract=off reference:
 *   - this translation unit is compiled with -fmad=false -prec-div=true -prec-sqrt=true -ftz=false
 *     (see __graft_entry__.build); every a*b+c therefore rounds twice exactly like the CPU build;
 *   - min/max/clamp are the TERNARY macros of includes.h:20-21 (NaN behaviour differs from fminf);
 *   - libm calls (sinf cosf powf atan2f acosf asinf logf fmodf) are evaluated in fp64 and rounded
 *     once to fp32: glibc's fp32 routines are correctly rounded in all but a vanishing fraction of
 *     inputs, and so is this (measured effect on the image: RMSE ~3e-7, SURVEY.md App. C).
 */
#pragma once
#include <stdint.h>
#include <cuda_runtime.h>

#define CR_PI 3.141592653589793238462643383279502f /* includes.h:13 */
#define CR_MIN(a, b) (((a) < (b)) ? (a) : (b))
#define CR_MAX(a, b) (((a) > (b)) ? (a) : (b))
#define CR_FLT_MAX 3.402823466e+38f

#define CRD __device__ __forceinline__

struct v3 { float x, y, z; };
struct v2 { float x, y; };
struct col3 { float r, g, b; };       /* the alpha lane of struct color never reaches the framebuffer */
struct col4 { float r, g, b, a; };


/* ---- libm stand-ins: fp64 evaluation, one rounding ------------------------------------------------
 * __noinline__ on purpose: each is a few hundred SASS instructions of fp64 code; one shared copy keeps
 * the shade kernel small (i-cache) and the build fast. */
#define CRN static __device__ __noinline__
CRN float cr_sinf(float x) { return (float)sin((double)x); }
CRN float cr_cosf(float x) { return (float)cos((double)x); }
CRN float2 cr_sincosf2(float x) { double ds, dc; sincos((double)x, &ds, &dc); return make_float2((float)ds, (float)dc); }
CRD void cr_sincosf(float x, float *s, float *c) { const float2 r = cr_sincosf2(x); *s = r.x; *c = r.y; }
/* powf(x, y): fp64 evaluation rounded once.  For x > 0 it is exp(y*log(x)) (relative error ~1e-15, i.e. the
 * fp32 result differs from the correctly rounded one for ~1e-8 of inputs — glibc's own powf is off more often);
 * everything else (zero, negative, inf, nan) goes through the full pow() special-case logic. */
CRN float cr_powf(float x, float y) {
	if (x > 0.0f && x < CR_FLT_MAX && y == y && fabsf(y) < 1.0e6f) return (float)exp((double)y * log((double)x));
	return (float)pow((double)x, (double)y);
}
/* powf(x, 5.0f) as used by schlick() (vector.h:271): four fp64 products, one rounding */
CRD float cr_pow5f(float x) { const double a = (double)x, a2 = a * a; return (float)(a2 * a2 * a); }
CRN float cr_logf(float x) { return (float)log((double)x); }
CRN float cr_log10f(float x) { return (float)log10((double)x); }     /* math.c:66 */
CRN float cr_tanf(float x) { return (float)tan((double)x); }         /* math.c:87 */
CRN float cr_atan2f(float y, float x) { return (float)atan2((double)y, (double)x); }
CRN float cr_acosf(float x) { return (float)acos((double)x); }
CRN float cr_asinf(float x) { return (float)asin((double)x); }
CRD float cr_fmodf(float x, float y) { return fmodf(x, y); }   /* fmodf is exact in any correct libm */
CRD float cr_sqrtf(float x) { return __fsqrt_rn(x); }
CRD float cr_div(float a, float b) { return __fdiv_rn(a, b); }

/* ---- vector.h ---------------------------------------------------------------------------------------- */
CRD v3 v3make(float x, float y, float z) { v3 r; r.x = x; r.y = y; r.z = z; return r; }
CRD v3 v3add(v3 a, v3 b) { return v3make(a.x + b.x, a.y + b.y, a.z + b.z); }                 /* :65 */
CRD v3 v3sub(v3 a, v3 b) { return v3make(a.x - b.x, a.y - b.y, a.z - b.z); }                 /* :76 */
CRD v3 v3mul(v3 a, v3 b) { return v3make(a.x * b.x, a.y * b.y, a.z * b.z); }                 /* :80 */
CRD float v3dot(v3 a, v3 b) { return a.x * b.x + a.y * b.y + a.z * b.z; }                    /* :91 */
CRD v3 v3scale(v3 v, float c) { return v3make(v.x * c, v.y * c, v.z * c); }                  /* :102 */
CRD v3 v3cross(v3 a, v3 b) {                                                                 /* :121 */
	return v3make((a.y * b.z) - (a.z * b.y), (a.z * b.x) - (a.x * b.z), (a.x * b.y) - (a.y * b.x));
}
CRD float v3len(v3 v) { return cr_sqrtf(v3dot(v, v)); }                                      /* :162 */
CRD v3 v3norm(v3 v) { float l = v3len(v); return v3make(cr_div(v.x, l), cr_div(v.y, l), cr_div(v.z, l)); } /* :173 */
CRD v3 v3neg(v3 v) { return v3make(-v.x, -v.y, -v.z); }
CRD v3 v3reflect(v3 I, v3 N) { return v3sub(I, v3scale(N, v3dot(N, I) * 2.0f)); }            /* :211 */
CRD float cr_clamp(float value, float lo, float hi) { return CR_MIN(CR_MAX(value, lo), hi); } /* :55 */
CRD float cr_wrapMax(float x, float mx) { return cr_fmodf(mx + cr_fmodf(x, mx), mx); }        /* :215 */
CRD float cr_wrapMinMax(float x, float mn, float mx) { return mn + cr_wrapMax(x - mn, mx - mn); } /* :219 */

/* ---- color.h --------------------------------------------------------------------------------------------- */
CRD col4 c4make(float r, float g, float b, float a) { col4 c; c.r = r; c.g = g; c.b = b; c.a = a; return c; }
CRD col4 c4add(col4 a, col4 b) { return c4make(a.r + b.r, a.g + b.g, a.b + b.b, a.a + b.a); }   /* :38 */
CRD col4 c4coef(float k, col4 c) { return c4make(c.r * k, c.g * k, c.b * k, c.a * k); }         /* :49 */
CRD col4 c4mix(col4 a, col4 b, float t) { return c4add(c4coef(1.0f - t, a), c4coef(t, b)); }    /* :54 */
CRD float cr_srgb_to_linear(float c) {                                                          /* :68 */
	if (c <= 0.04045f) return cr_div(c, 12.92f);
	return cr_powf(cr_div(c + 0.055f, 1.055f), 2.4f);
}
CRD float cr_linear_to_srgb(float c) {                                                          /* :60 */
	if (c <= 0.0031308f) return 12.92f * c;
	return (1.055f * cr_powf(c, 0.4166666667f)) - 0.055f;
}
CRD float cr_grayscale(col4 c) {                                                                /* :43, double constants */
	double sum = (double)(0.299f * cr_powf(c.r, 2.0f)) + 0.587 * (double)cr_powf(c.g, 2.0f) + 0.114 * (double)cr_powf(c.b, 2.0f);
	return cr_sqrtf((float)sum);
}
static __device__ __noinline__ col4 cr_color_for_kelvin(float kelvin) {                                                    /* color.c:28-70 */
	float r, g, b;
	float temp = kelvin >= 40000.0f ? 40000.0f : kelvin;
	temp = cr_div(temp, 100.0f);
	if (temp <= 66.0f) {
		r = 255.0f;
	} else {
		r = temp - 60.0f;
		r = 329.698727446f * cr_powf(r, -0.1332047592f);
		r = r < 0.0f ? 0.0f : r;
		r = r > 255.0f ? 255.0f : r;
	}
	if (temp <= 66.0f) {
		g = temp;
		g = 99.4708025861f * cr_logf(g) - 161.1195681661f;
		g = g < 0.0f ? 0.0f : g;
		g = g > 255.0f ? 255.0f : g;
	} else {
		g = temp - 60.0f;
		g = 288.1221695283f * cr_powf(g, -0.0755148492f);
		g = g < 0.0f ? 0.0f : g;
		g = g > 255.0f ? 255.0f : g;
	}
	if (temp >= 66.0f) {
		b = 255.0f;
	} else if (temp <= 19.0f) {
		b = 0.0f;
	} else {
		b = temp - 10.0f;
		b = 138.5177312231f * cr_logf(b) - 305.0447927307f;
		b = b < 0.0f ? 0.0f : b;
		b = b > 255.0f ? 255.0f : b;
	}
	return c4make(cr_div(r, 255.0f), cr_div(g, 255.0f), cr_div(b, 255.0f), 0.0f);
}

/* ---- transforms.c:76-116 (row-major 4x4, only the top three rows are ever read) --------------------------- */
CRD v3 xf_point(const float *m, v3 v) {
	return v3make((m[0] * v.x) + (m[1] * v.y) + (m[2] * v.z) + m[3],
				  (m[4] * v.x) + (m[5] * v.y) + (m[6] * v.z) + m[7],
				  (m[8] * v.x) + (m[9] * v.y) + (m[10] * v.z) + m[11]);
}
CRD v3 xf_vector(const float *m, v3 v) {
	return v3make((m[0] * v.x) + (m[1] * v.y) + (m[2] * v.z),
				  (m[4] * v.x) + (m[5] * v.y) + (m[6] * v.z),
				  (m[8] * v.x) + (m[9] * v.y) + (m[10] * v.z));
}
CRD v3 xf_vector_transpose(const float *m, v3 v) {                                            /* :106-111 */
	return v3make((m[0] * v.x) + (m[4] * v.y) + (m[8] * v.z),
				  (m[1] * v.x) + (m[5] * v.y) + (m[9] * v.z),
				  (m[2] * v.x) + (m[6] * v.y) + (m[10] * v.z));
}

/* ---- sampler: common.h:22-27, pcg_basic.c:42-68, random.c:16-21; inc is always 1 -------------------------- */
CRD uint64_t cr_hash64(uint64_t x) {
	x = (x ^ (x >> 30)) * 0xbf58476d1ce4e5b9ull;
	x = (x ^ (x >> 27)) * 0x94d049bb133111ebull;
	x = x ^ (x >> 31);
	return x;
}
CRD uint32_t cr_pcg32(uint64_t &state) {
	uint64_t old = state;
	state = old * 6364136223846793005ull + 1ull;
	uint32_t xorshifted = (uint32_t)(((old >> 18u) ^ old) >> 27u);
	uint32_t rot = (uint32_t)(old >> 59u);
	return (xorshifted >> rot) | (xorshifted << ((0u - rot) & 31u));
}
CRD uint64_t cr_rng_init(uint32_t pixIdx, uint32_t pass, uint32_t maxPasses) {                /* sampler.c:41-44 */
	uint32_t seed32 = pixIdx * maxPasses + pass;   /* wraps in 32 bits, like the reference */
	uint64_t seed = cr_hash64((uint64_t)seed32);
	uint64_t state = 0ull;
	cr_pcg32(state);
	state += seed;
	cr_pcg32(state);
	return state;
}
CRD float cr_draw(uint64_t &state) {                                                          /* random.c:17 */
	return 2.3283064365386963e-10f * __uint2float_rn(cr_pcg32(state));   /* 2^-32 * (float)u32; can be 1.0f */
}

CRD v3 cr_random_on_unit_sphere(uint64_t &rng) {                                              /* vector.h:243-249 */
	const float sx = cr_draw(rng);
	const float sy = cr_draw(rng);
	const float a = sx * (2.0f * CR_PI);
	const float s = 2.0f * cr_sqrtf(CR_MAX(0.0f, sy * (1.0f - sy)));
	float sn, cs;
	cr_sincosf(a, &sn, &cs);
	return v3make(cs * s, sn * s, 1.0f - 2.0f * sy);
}

/* x86-64 cvttss2si semantics for (int)float and (size_t)float as GCC compiles them (texture.c:66-73) */
CRD int cr_f2i(float x) {
	if (!(x > -2147483904.0f && x < 2147483648.0f)) return (int)0x80000000;
	return __float2int_rz(x);
}
CRD uint64_t cr_f2sz(float x) {
	if (x < 9223372036854775808.0f) {
		if (!(x > -9223373136366403584.0f)) return 0x8000000000000000ull;
		return (uint64_t)__float2ll_rz(x);
	}
	if (!(x < 18446744073709551616.0f)) return 0x8000000000000000ull ^ 0x8000000000000000ull;
	return ((uint64_t)__float2ll_rz(x - 9223372036854775808.0f)) ^ 0x8000000000000000ull;
}

/* colorToSRGB + setPixel(char_p) of one channel: renderer.c:297-300, texture.c:19-21 */
CRD uint8_t cr_to_srgb8(float v) {
	const float c = cr_linear_to_srgb(v);
	const float s = CR_MIN(c * 255.0f, 255.0f);
	/* (unsigned char) of a negative/NaN float is UB in C; x86 cvttss2si + truncation gives the low byte */
	return (uint8_t)(cr_f2i(s) & 0xff);
}
