/*
 * crgpu_wave.cuh — wavefront buffers and kernel launchers shared by the translation units of libcrgpu.so.
 *
 * One `crgpu_render_tile` call processes a tile rectangle in batches of B passes; a batch has
 * N = tile_pixels * B paths, path id = p_local * tile_pixels + pixel_local.  Per batch:
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

struct TileDesc {
	int x0, y0, tw, th;     /* tile origin and size (pixels); y up */
	int pass_begin, pass_count; /* this batch */
	const uint32_t *pixels; /* NULL: the pixel set is the rectangle above; else an explicit list x | y << 16 (a union of tiles) */
	unsigned npix;          /* number of pixels in the set */
};

__device__ __forceinline__ void crg_pixel_xy(const TileDesc &td, unsigned px, int &x, int &y) {
	if (td.pixels) { const uint32_t p = __ldg(td.pixels + px); x = (int)(p & 0xffffu); y = (int)(p >> 16); }
	else { x = td.x0 + (int)(px % (unsigned)td.tw); y = td.y0 + (int)(px / (unsigned)td.tw); }
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
void crg_launch_pixel_list(uint32_t *pixels, const int4 *rects, const unsigned *offs, int nrects, cudaStream_t st);
void crg_launch_generate(const DevScene &sc, const WaveBuffers &wb, const TileDesc &td, int grid, cudaStream_t st);
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
/* gate: NULL, or the stop words of an armed scene (below): K5 then adds the batch only if wave set `set`'s batch was not abandoned
 * and the committed pass index equals td.pass_begin.  snap_host: NULL, or (a batch that publishes) the host words, whose snapshot
 * state K5 reads once into gate[3] for the publish step */
void crg_launch_accumulate(float *fb, const float4 *L, const TileDesc &td, int W, int H, int grid, cudaStream_t st,
                           unsigned *gate = nullptr, int set = 0, const unsigned *snap_host = nullptr);

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
