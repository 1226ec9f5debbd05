/*
 * crgpu_wave.cuh — wavefront buffers and kernel launchers shared by the translation units of libcrgpu.so.
 *
 * One `crgpu_render_tile` call processes a tile rectangle in batches of B passes; a batch has
 * N = tile_pixels * B paths, numbered by the path order (crg_path_pass_pixel below; pass-major, id = p_local * tile_pixels +
 * pixel_local, with CRGPU_PATH_ORDER=0).  Per batch:
 *
 *   K1 k_generate    initSampler + getCameraRay for every path            (sampler.c:41-44, camera.c:58-87)
 *   per bounce:
 *   K2 k_trace       closest hit of every live ray                        (pathtrace.c:38 → bvh.c, poly.c, sphere.c)
 *   K4 k_bucket      counting sort of the live rays by shading bucket (miss / material id) so that the
 *                    32 lanes of a K3 warp run the same node graph (K2 fills the histogram)
 *   K3 k_shade       miss → background, hit → emission, bsdf sample, Russian roulette, weight update;
 *                    survivors are COMPACTED into the other half of the ping-pong ray buffers with one
 *                    warp-ballot + one atomicAdd per warp (K4 is fused into K3)   (pathtrace.c:39-57)
 *   K5 k_accumulate  running average of the B pass samples into the fp32 framebuffer, in pass order
 *                                                                         (renderer.c:288-294)
 *
 * Path state in HBM (SoA of 16-byte vectors, always read/written at the COMPACT live index, so every
 * access is a coalesced 128-bit transaction):
 *   stA = (o.x, o.y, o.z, d.x)   stB = (d.y, d.z, weight.r, weight.g)   stC = (weight.b, path id, rng lo, rng hi)
 *   hit = (t, u, v, prim slot)   hitInst = instance index or -1
 *   L[path id] = (r, g, b, -)    radiance of the path, written at termination / emissive hits
 * The queue order never affects results: every path carries its own RNG state and id.
 */
#pragma once
#include <cuda_runtime.h>
#include "crgpu_scene.cuh"

struct WaveBuffers {
	float4 *stA[2];
	float4 *stB[2];
	uint4  *stC[2];
	float4 *hit;
	int    *hitInst;
	float4 *L;
	unsigned char *hitKey;  /* shading bucket of the hit: 0 = miss, else min(material+1, 255) */
	unsigned *perm;         /* K4 output: live indices grouped by bucket */
	unsigned char *dirKey;  /* direction bin of every ray K3 wrote for the next bounce (crg_dir_mode) */
	unsigned *perm2;        /* K4b output: the next bounce's rays grouped by direction bin — the order K2 hands them to its lanes */
	unsigned *hist;         /* [256] bucket sizes (filled by K2), [256..511] K4 cursors, [512..767] direction-bin sizes (filled by K3),
	                           [768..1023] K4b cursors */
	unsigned *counts;       /* [0],[1]: live counts of the ping-pong halves; [2]: K2's work counter (next ray to hand out); [3]: tail-kernel block counter; [4]: number of misses of this bounce (K4 -> K3 split); [5]: end of the flat materials' range of perm (K4 -> K3 flat launch) */
	unsigned *box;          /* [CRG_BOX_SLOTS][12]: bounds of the origins K3 wrote at depth min(d, CRG_BOX_SLOTS - 1), for the origin cell of
	                           dir mode 4.  [0..5] = this batch (lo x,y,z as ~crg_ord(lo), hi x,y,z as crg_ord(hi); atomicMax, 0 = empty),
	                           [6..11] = the previous batch of this wave set: K3 keys its rays with those, K4b moves [0..5] there */
	unsigned long long *stats; /* [0] rays, [1] pairs, [2] tris, [3] spheres, [4] insts, [5] paths committed by armed calls,
	                              [7] traversal watchdog */
};

/* Half h of a ping-pong state array.  Indexing the kernel-parameter array (wb.stA[cur]) with a runtime value makes the compiler
 * copy the whole WaveBuffers parameter to local memory at kernel entry and reload every wb.* pointer from there; selecting
 * between the two members keeps the parameter in the constant bank.  ptxas -v, stack frame / spill stores with the copy and
 * without: k_trace<false,3,0> 768 B / 186 B and 568 B / 110 B; K3's hit kernel (k_shade<2,2,false>) 416 B / 124 B and 304 B / 170 B. */
template <class T> __device__ __forceinline__ T *crg_half(T *const (&a)[2], int h) { return h ? a[1] : a[0]; }

/* The host words of an armed scene are pinned, mapped memory: read and written at system scope, so a host store is seen by the next
 * kernel that reads it and a device store by the host without any synchronisation. */
__device__ __forceinline__ unsigned crg_ld_sys(const unsigned *p) {
	unsigned v;
	asm volatile("ld.relaxed.sys.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
	return v;
}
__device__ __forceinline__ void crg_st_sys(unsigned *p, unsigned v) { asm volatile("st.relaxed.sys.global.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory"); }

/* ---- path order (CRGPU_PATH_ORDER, crg_path_order) ---------------------------------------------------------------------------
 * K2 hands rays to its lanes in path-id order at bounce 0, and K3's compaction keeps that order within a material bucket for the
 * bounces after, so the order in which a batch numbers its (pass, pixel) pairs decides which rays share a warp.  Two choices:
 *   blocked  the pixels of a rectangle (a tile of a tile list, or the rectangle of crgpu_render_tile) are numbered in 8x4 blocks,
 *            Morton order inside a block (crg_block_xy), instead of row by row;
 *   P, Q     the passes are taken in groups of P, and inside a group the paths run over Q consecutive pixels for each of the
 *            group's passes before the next Q pixels (crg_path_pass_pixel).  P = 1 is pass-major order.
 * With blocked pixels and P * Q = 32, the 32 lanes a warp refills at bounce 0 trace P passes of one 2D block of Q pixels. */
struct PathOrder { unsigned p, q; int blocked; };
/* the values of CRGPU_PATH_ORDER: 0 = pass-major over row-by-row pixels (the order before the knob existed); 1 = pass-major over
 * 8x4 pixel blocks; 2, 3, 4 = 8, 4, 2 passes of one 2x2, 4x2, 4x4 pixel block per 32 paths; 5 = 8 passes of a 4x1 strip of
 * row-by-row pixels; 6 = 16 passes of a 2x1 pair of blocked pixels; 7 = 32 passes of one pixel (pixels in blocked order) */
#define CRG_PATH_ORDERS 8
inline PathOrder crg_path_order_of(int v) {
	static const PathOrder t[CRG_PATH_ORDERS] = { { 1u, 32u, 0 }, { 1u, 32u, 1 }, { 8u, 4u, 1 }, { 4u, 8u, 1 }, { 2u, 16u, 1 }, { 8u, 4u, 0 },
	                                              { 16u, 2u, 1 }, { 32u, 1u, 1 } };
	return t[v];
}
const PathOrder &crg_path_order(void);     /* the frame path's order, CRGPU_PATH_ORDER (crgpu_trace.cu) */

/* pixel i of a w x h rectangle in blocked order: the whole 8x4 blocks row of blocks by row of blocks, Morton order inside a block
 * (bits x0 y0 x1 y1 x2: 4, 8, 16 and 32 aligned consecutive pixels are 2x2, 4x2, 4x4 and 8x4 squares), then the pixels right of
 * the whole blocks row by row, then the rows below them.  A bijection of [0, w*h) for every w, h >= 1. */
__host__ __device__ __forceinline__ void crg_block_xy(unsigned i, unsigned w, unsigned h, unsigned &x, unsigned &y) {
	const unsigned bw = w >> 3, bh = h >> 2, inner = bw * bh * 32u;
	if (i < inner) {
		const unsigned b = i >> 5, m = i & 31u, by = b / bw, bx = b - by * bw;
		x = (bx << 3) | (m & 1u) | ((m >> 1) & 2u) | ((m >> 2) & 4u);
		y = (by << 2) | ((m >> 1) & 1u) | ((m >> 2) & 2u);
		return;
	}
	const unsigned r = i - inner, rw = w - (bw << 3), right = rw * (bh << 2);
	if (r < right) { y = r / rw; x = (bw << 3) + (r - y * rw); return; }
	const unsigned r2 = r - right;
	y = (bh << 2) + r2 / w; x = r2 - (y - (bh << 2)) * w;
}

/* the path order of a batch of npix pixels and pass_count passes (P = o.p, Q = o.q): pass group c holds passes [cP, cP + Pc),
 * Pc = min(P, pass_count - cP), and paths [cP * npix, (cP + Pc) * npix); inside it the whole blocks of Q pixels come first, each
 * as Pc runs of Q paths (one run per pass), then the last npix mod Q pixels as Pc runs of that many.  A bijection of
 * [0, npix * pass_count) onto (pass_local, pixel_local) for every npix, pass_count >= 1 (checked on the host through crgpu_path_order_map). */
__host__ __device__ __forceinline__ void crg_path_pass_pixel(unsigned id, unsigned npix, unsigned pass_count, unsigned P, unsigned Q,
                                                            unsigned &pl, unsigned &px) {
	const unsigned c0 = (id / npix) / P * P;                                  /* = floor(id / (P npix)) * P without the product */
	const unsigned pc = pass_count - c0 < P ? pass_count - c0 : P;
	const unsigned r = id - c0 * npix, h = npix / Q, full = pc * Q * h;
	if (r < full) {
		const unsigned run = pc * Q, b = r / run, k = r - b * run, j = k / Q;
		pl = c0 + j; px = b * Q + (k - j * Q);
	} else {
		const unsigned s = npix - Q * h, r2 = r - full, j = r2 / s;
		pl = c0 + j; px = Q * h + (r2 - j * s);
	}
}
/* the inverse: the path id of (pass_local, pixel_local) */
__host__ __device__ __forceinline__ unsigned crg_path_id(unsigned pl, unsigned px, unsigned npix, unsigned pass_count, unsigned P, unsigned Q) {
	const unsigned c0 = pl / P * P, pc = pass_count - c0 < P ? pass_count - c0 : P, j = pl - c0, h = npix / Q;
	if (px < Q * h) { const unsigned b = px / Q; return c0 * npix + b * pc * Q + j * Q + (px - b * Q); }
	return c0 * npix + pc * Q * h + j * (npix - Q * h) + (px - Q * h);
}

struct TileDesc {
	int x0, y0, tw, th;     /* tile origin and size (pixels); y up */
	int pass_begin, pass_count; /* this batch */
	const uint32_t *pixels; /* NULL: the pixel set is the rectangle above; else an explicit list x | y << 16 (a union of tiles) */
	unsigned npix;          /* number of pixels in the set */
	PathOrder order;        /* how the batch numbers its paths (set by render_batches) */
};

__device__ __forceinline__ void crg_pixel_xy(const TileDesc &td, unsigned px, int &x, int &y) {
	if (td.pixels) { const uint32_t p = __ldg(td.pixels + px); x = (int)(p & 0xffffu); y = (int)(p >> 16); }
	else if (td.order.blocked) { unsigned bx, by; crg_block_xy(px, (unsigned)td.tw, (unsigned)td.th, bx, by); x = td.x0 + (int)bx; y = td.y0 + (int)by; }
	else { x = td.x0 + (int)(px % (unsigned)td.tw); y = td.y0 + (int)(px / (unsigned)td.tw); }
}

/* ---- several views in one call (crgpu_render_views) ---------------------------------------------------------------------------
 * A views call numbers its (view, pixel) pairs view-major: call pixel g is view view0 + g / npix at pixel g mod npix of the tile
 * set's pixel list (TileDesc::pixels, never a rectangle).  A piece is the range [p0, p0 + TileDesc::npix) of that numbering, and
 * the path order maps a batch's ids onto (pass, piece pixel) exactly as for one view.  Only K1 (the camera) and K5 (the framebuffer)
 * look at the view; they are launched in their <VIEWS = true> instantiations.  The camera of view 0 is the scene's (cam0: the HBM
 * copy of DevScene::cam, which every edit publishes), its framebuffer the scene's. */
struct ViewDesc {
	const DevCamera *cam0;  /* view 0's camera */
	const DevCamera *cams;  /* views 1..: view v's camera is cams[v - 1] */
	float *fb;              /* views 1..: view v's framebuffer is fb + (v - 1) * fb_floats */
	size_t fb_floats;
	unsigned npix;          /* pixels of the tile set (per view) */
	unsigned view0;         /* the call's first view */
	unsigned p0;            /* the piece's first call pixel */
};
/* view and tile-set pixel of piece pixel px */
__device__ __forceinline__ void crg_view_pixel(const ViewDesc &vd, unsigned px, unsigned &v, unsigned &tp) {
	const unsigned g = vd.p0 + px, q = g / vd.npix;
	v = vd.view0 + q; tp = g - q * vd.npix;
}

/* Launch variant of K2.  Every variant computes the same hit records; they differ in how a warp schedules its work.
 *   minb      blocks per SM the compiler makes room for: 2, 3 or 4 (the instrumented kernel, count = true, always uses 3)
 *   defer     0 = leaf triangles tested inside the node step, 1 = after the node burst by each lane, 2 = dealt over the warp
 *   refill    a warp fetches new rays when fewer than `refill` lanes are busy (1..32)
 *   burst     child-pair steps per node phase (>= 1)
 *   inst_min  lanes that must want an instance step before the warp takes one (1..32)
 * The frame path reads them once from CRGPU_TRACE_MINB / _DEFER / _REFILL / _BURST / _INSTMIN (crg_trace_knobs_env);
 * crgpu_trace_rays passes its own. */
struct TraceKnobs { int minb, defer, refill, burst, inst_min; };
const TraceKnobs &crg_trace_knobs_env(void);

/* launchers (defined in crgpu_trace.cu / crgpu_shade.cu); `dsc` is the device copy of `sc` */
void crg_launch_pixel_list(uint32_t *pixels, const int4 *rects, const unsigned *offs, int nrects, int blocked, cudaStream_t st);
/* vd: NULL, or the views of a views call (K1 <VIEWS = true>) */
void crg_launch_generate(const DevScene &sc, const WaveBuffers &wb, const TileDesc &td, const ViewDesc *vd, int grid, cudaStream_t st);
void crg_launch_trace(const DevScene &sc, const WaveBuffers &wb, int cur, bool count, bool sorted, const TraceKnobs &kn, cudaStream_t st);
/* per-ray records of K2's write-back (crgpu_trace_rays): t, u, v, instance, poly (-1 for spheres and misses), key */
void crg_launch_trace_records(const DevScene &sc, const WaveBuffers &wb, unsigned n, void *out, int grid, cudaStream_t st);
#define CRG_BOX_SLOTS 32
/* box_slot: the depth slot whose bounds K4b moves to the previous-batch half (dir mode 4), or -1 */
void crg_launch_dirsort(const WaveBuffers &wb, int nxt, int box_slot, int grid, cudaStream_t st);
/* 0 = off, 1 = octant (8 bins), 2 = octant x major axis (24 bins), 3 = octant x origin cell in the world box (256 bins),
 * 4 = octant x 5-bit Morton cell of the origin in the bounds of the previous batch's origins at the same depth (256 bins) */
int crg_dir_mode(void);
/* K4.  order: NULL (buckets in key order) or DevScene::key_order with nflat = DevScene::flat_keys (the flat materials' buckets
 * right behind the misses, for the flat K3 launch); it also writes counts[4] (misses) and counts[5] (end of the flat range) */
void crg_launch_bucket(const WaveBuffers &wb, int cur, int grid, const uint8_t *order, int nflat, cudaStream_t st);
void crg_launch_tail(const DevScene *dsc, const WaveBuffers &wb, int cur, int depth, int maxDepth, bool xnodes, cudaStream_t st);
/* Launch variant of K3.  Every variant computes the same path states.
 *   minb          blocks per SM of the generic hit kernel (or of the one kernel when not split): 2, 3 or 4
 *   split         1 = a separate miss kernel (PART 1) ahead of the hit kernels (PART 3, PART 2); 0 = one kernel for every ray (PART 0)
 *   prefetch      1 = read perm two iterations ahead and prefetch the records it points to into L2
 *   generic_only  1 = no flat launch: every hit goes through the node interpreter (PART 2), K4 keeps the buckets in key order
 *   flat_minb     blocks per SM of the flat hit kernel (PART 3): 2, 3 or 4
 * The frame path reads them once from CRGPU_SHADE_MINB / _SPLIT / _PREFETCH / _GENERIC_ONLY / _FLAT_MINB (crg_shade_knobs_env);
 * crgpu_shade_rays passes its own. */
struct ShadeKnobs { int minb, split, prefetch, generic_only, flat_minb; };
const ShadeKnobs &crg_shade_knobs_env(void);
/* flat_bg: DevScene::bg is folded (the miss launch samples it inline).  ev: NULL, or three events recorded after the miss, the flat
 * and the generic launch (CRGPU_FLAG_TIME_KERNELS' per-launch split).  Returns the number of kernels it launched.  The bounce
 * sequence around it (K2, K4, this, K4b) is enqueue_bounce in crgpu_api.cu, for the frame and for crgpu_shade_rays alike. */
int crg_launch_shade(const DevScene *dsc, const WaveBuffers &wb, int cur, int depth, int maxDepth, int dirmode, bool xnodes, bool flat_bg, int grid,
                     const ShadeKnobs &kn, cudaStream_t st, cudaEvent_t *ev);
/* whether K4 must order the buckets for the flat launch (crg_launch_bucket's order) */
bool crg_shade_flat_order(const ShadeKnobs &kn);
/* the libm stand-ins of crgpu_math.cuh one by one (crgpu_libm_eval) */
void crg_launch_libm(int fn, const float *x, const float *y, float *out, unsigned n, cudaStream_t st);
/* ---- adaptive rounds (crgpu_adaptive_round) -------------------------------------------------------------------------------------
 * Every pixel of view 0 has one record, at its framebuffer index (x + (H - 1 - y) W): the passes its framebuffer holds, the Welford
 * mean and M2 of their luminance, and the error of its last convergence test.  Only K5 <ADAPTIVE> adds passes to a record, and only
 * passes it commits; the select kernels test and mark pixels done. */
#define CRG_ADAPT_DONE 0x80000000u   /* AdaptPix::n: the pixel has converged */
struct AdaptPix { uint32_t n; float mean, m2, err; };
struct AdaptParams { unsigned min_passes, round_passes, pass_end; float threshold, floor; };
/* every record of n to { 0, 0, 0, +inf } */
void crg_launch_adapt_reset(AdaptPix *recs, size_t n, cudaStream_t st);
/* select, step 1 of 2: for pixel i of the list (x | y << 16), whether it stays active after the test at its count (flags[i] = 0 or 1),
 * and into mm the max of ~n and of n over the active pixels (mm zeroed before) */
void crg_launch_adapt_select(const uint32_t *pixels, unsigned npix, const AdaptPix *recs, int W, int H, const AdaptParams &a,
                             unsigned long long *flags, unsigned *mm, cudaStream_t st);
/* step 2, after the inclusive scan incl of flags: when every active pixel has the same count (or none is active) each tested pixel
 * takes its error and done bit and each active pixel its place in the active list; in any case host[0..2] = active count, min and
 * max count */
void crg_launch_adapt_compact(const uint32_t *pixels, unsigned npix, AdaptPix *recs, int W, int H, const AdaptParams &a,
                              const unsigned long long *flags, const unsigned long long *incl, uint32_t *active, const unsigned *mm,
                              unsigned *host, cudaStream_t st);

/* gate: NULL, or the stop words of an armed scene (below): K5 then adds the batch only if wave set `set`'s batch was not abandoned
 * and the committed pass index equals td.pass_begin.  snap_host: NULL, or (a batch that publishes) the host words, whose snapshot
 * state K5 reads once into gate[3] for the publish step.  vd: NULL, or the views of a views call (K5 <ARMED, VIEWS = true>: each
 * (view, pixel) into its view's framebuffer; armed, it clears gate[3], so a views call never stages a snapshot).  adapt: NULL, or
 * the records of an adaptive round (K5 <ADAPTIVE = true>, never with vd): each added pass also updates its pixel's record. */
void crg_launch_accumulate(float *fb, const float4 *L, const TileDesc &td, int W, int H, int grid, cudaStream_t st,
                           unsigned *gate = nullptr, int set = 0, const unsigned *snap_host = nullptr, const ViewDesc *vd = nullptr,
                           AdaptPix *adapt = nullptr);

/* ---- stopping an armed scene at a pass boundary (crgpu_stop_enable) ----------------------------------------------------------------
 * ctl (device memory): [0] the pass index the running average has reached in this call, [1 + set] wave set `set`'s batch was
 * abandoned, [3] the publish step stages a snapshot (written by K5), [4] the publish step's count of finished blocks.
 * host (pinned, mapped): [0] stop request, [1] committed pass index (published), [2] a call is in flight, [3] snapshot state
 * (0 idle, 1 requested, 2 staged), [4] the pass index of the staged snapshot.
 * The gate runs after K1 and before every bounce; if the stop is requested (and `check`) it abandons the batch and leaves the wave
 * set as k_tail leaves it, so the rest of the batch's kernels run on zero rays.  `reset`: the first gate of a batch.  No kernel
 * waits for the host: pausing is the host's business. */
void crg_launch_stop_gate(unsigned *counts, int cur, unsigned *ctl, int set, const unsigned *host, bool reset, bool check, cudaStream_t st);
void crg_launch_stop_begin(unsigned *ctl, unsigned *host, int pass_begin, cudaStream_t st);
/* after K5: advance ctl[0] past the batch if K5 added it (and count its paths in stats[5]), then publish ctl[0].  When K5 found a
 * snapshot requested (ctl[3]), the grid also converts the whole framebuffer fb (n floats) to sRGB8 into snap, and its last block
 * publishes ctl[0] as the snapshot's pass index and sets the state to staged.  Otherwise every block but the first returns at once. */
void crg_launch_stop_publish(unsigned *ctl, int set, unsigned *host, int pass_begin, int pass_count, unsigned long long paths,
                             unsigned long long *stats, const float *fb, uint8_t *snap, size_t n, int grid, cudaStream_t st);
/* the call's last kernel: publish ctl[0] and clear the in-flight word */
void crg_launch_stop_end(unsigned *ctl, unsigned *host, cudaStream_t st);
void crg_launch_to_srgb8(const float *fb, uint8_t *out, size_t n, int grid, cudaStream_t st);
void crg_launch_kat(const DevScene *dsc, const int32_t *xyp, int count, void *out, cudaStream_t st);
