/*
 * crgpu.h — C ABI of the H100 path-trace hot loop (libcrgpu.so).
 *
 * This is the drop-in boundary.  c-ray's tile dispatcher (`renderFrame`, reference
 * src/renderer/renderer.c:40-180) starts worker threads through a `struct crThread` slot whose
 * `threadFunc` is today `renderThread` (renderer.c:258-327) or `networkRenderThread`
 * (src/utils/protocol/server.c:215-263).  A GPU worker thread occupies the same slot
 * (c-ray_b200/host/cr_renderer.c `gpuRenderThread`; the reference-side binding is c-ray_b200/integration/gpu_thread.c, INTEGRATION.md) and calls ONLY the functions
 * below — plain pointers and sizes, no CUDA or torch types.
 *
 *   reference interface replaced                                  entry point here
 *   -----------------------------------------------------------   ---------------------------------
 *   (none; scene is read through pointers, scene.h:14-39)          crgpu_scene_create / _destroy
 *   renderThread inner loops, renderer.c:271-320                   crgpu_render_tile
 *     initSampler  sampler.c:41-44   getCameraRay camera.c:58-87
 *     pathTrace    pathtrace.c:32-60 traverseTopLevelBvh bvh.c:488
 *     bsdf->sample nodes/shaders     running average renderer.c:288-294
 *   colorToSRGB + setPixel(image), renderer.c:297-300              crgpu_framebuffer_to_srgb8
 *   textureGetPixel(renderBuffer), renderer.c:283                  crgpu_framebuffer_read / _write / _clear
 *   tile gather of the cluster mode, server.c:159-174              crgpu_framebuffer_device_ptr (+ NCCL in the host)
 *   buildBvhGeneric, src/accelerators/bvh.c:245-296                crgpu_bvh_build (SURVEY 8 f1; optional: the loaders build on the host)
 *
 * All functions return 0 on success or a negative CRGPU_ERR_* code; crgpu_last_error() gives text.
 * The host turns errors into logr(warning|error, ...) like the rest of c-ray (logging.c:50-74).
 * There is NO CPU fallback: without a CUDA device every call fails with CRGPU_ERR_NO_DEVICE.
 */
#pragma once
#include <stdint.h>
#include <stddef.h>
#include "crscene.h"

#ifdef __cplusplus
extern "C" {
#endif

#define CRGPU_OK                 0
#define CRGPU_ERR_NO_DEVICE     -1
#define CRGPU_ERR_CUDA          -2
#define CRGPU_ERR_BAD_ARGUMENT  -3
#define CRGPU_ERR_UNSUPPORTED   -4   /* node graph deeper than the device interpreter supports, etc. */
#define CRGPU_ERR_NOMEM         -5
#define CRGPU_STOPPED            1   /* not an error: an armed render call ended at a pass boundary because a stop was requested */
#define CRGPU_PENDING            2   /* not an error: the snapshot asked for has not been staged yet (crgpu_take_snapshot) */

typedef struct crgpu_scene crgpu_scene;

/* Per-call statistics (all counted on the device). */
struct crgpu_stats {
	uint64_t paths;          /* pixel-passes started (one pathTrace call each) */
	uint64_t rays;           /* closest-hit queries, one per getClosestIsect (pathtrace.c:38) */
	uint64_t node_pairs;     /* P: BVH child-pair steps, both levels   (only with CRGPU_FLAG_COUNT) */
	uint64_t tri_tests;      /* T: triangle tests                      (only with CRGPU_FLAG_COUNT) */
	uint64_t sphere_tests;   /* S: sphere tests                        (only with CRGPU_FLAG_COUNT) */
	uint64_t inst_visits;    /* I: mesh-instance visits                (only with CRGPU_FLAG_COUNT) */
	uint64_t kernel_launches;/* CUDA kernels launched by this call */
	float    trace_ms;       /* device time inside the BVH-traversal kernel (CUDA events), if CRGPU_FLAG_TIME_KERNELS */
	float    shade_ms;       /* device time inside the shade kernel, same condition */
	float    total_ms;       /* device time of the whole call on its stream, same condition */
	float    pad;
};

#define CRGPU_FLAG_COUNT         0x1u  /* run the instrumented traversal kernel (slower; fills P/T/S/I) */
#define CRGPU_FLAG_TIME_KERNELS  0x2u  /* bracket every kernel with CUDA events (adds sync at the end only) */
#define CRGPU_FLAG_ASYNC         0x4u  /* only enqueue on the scene's stream; fetch the numbers later with crgpu_get_stats */

int crgpu_device_count(int *n);
const char *crgpu_last_error(void);

/* Upload a flattened scene (include/crscene.h) to `device`.  The device keeps its own replicas; the
 * flat arrays may be freed after the call.  Also allocates the fp32 framebuffer (W*H*3, row H-1-y:
 * the layout of state.renderBuffer, scene.c:200 + texture.c:24-28), zero-initialised. */
int crgpu_scene_create(const struct crs_scene *flat, int device, crgpu_scene **out);
int crgpu_scene_destroy(crgpu_scene *s);

/* The two halves of crgpu_scene_create, for hosts that render many frames of one scene or one frame on several GPUs (the
 * reference rebuilds nothing between frames either: loadScene builds the BVHs once, scene.c:111-213).  crgpu_prepare
 * validates the flat scene and re-lays it out for the kernels into ONE pinned host slab (device-independent, host threads);
 * crgpu_scene_create_prepared is then a single host->device copy.  Image size / sample count / bounces / camera are taken
 * from the flat scene at prepare time; crgpu_prepared_update_config re-reads them (after crscene_set_config) without
 * repacking.  crgpu_prepared_slab exposes the slab bytes (what crosses PCIe per frame; tests pin their checksum). */
typedef struct crgpu_prepared crgpu_prepared;
int  crgpu_prepare(const struct crs_scene *flat, crgpu_prepared **out);
int  crgpu_prepared_update_config(crgpu_prepared *p, const struct crs_scene *flat);
int  crgpu_prepared_slab(const crgpu_prepared *p, const void **slab, size_t *bytes);
void crgpu_prepared_free(crgpu_prepared *p);
/* How the shading kernels will sample each material: kinds[i] = 0 for a generic material (the node interpreter), else the flat
 * leaf (1 diffuse, 2 metal, 3 glass, 4 emissive, 5 plastic over a diffuse) with flags[i] bit 0 = under the alpha wrapper, bit 1 =
 * the wrapper's alpha is an image, bit 2 = the leaf colour is an image.  Fills min(count, material count) entries. */
int  crgpu_prepared_materials(const crgpu_prepared *p, uint32_t *kinds, uint32_t *flags, uint32_t count, uint32_t *material_count);
/* How the miss launch will sample the background: *kind = 0 through the node interpreter, else folded at upload with a constant
 * strength and offset over a 1 constant, 2 image or 3 gradient colour. */
int  crgpu_prepared_background(const crgpu_prepared *p, uint32_t *kind);
/* The slab sections the traversal's instance step reads, valid while p lives: one 64-byte record per top-level primIndices entry
 * (the instance's Ainv rows as 12 floats; its index | 1 << 31 for a mesh | 1 << 30 when the step must read the mesh's BVH record,
 * which is when that BVH has at most one node or staged nodes; its ray offset; a sphere's radius or a mesh BVH's pair offset; a mesh
 * BVH's slot offset), and the instance (128 B) and BVH (60 B) records they are built from.  Lengths in bytes. */
int  crgpu_prepared_top_level(const crgpu_prepared *p, const void **items, size_t *item_bytes, const void **instances,
                              size_t *instance_bytes, const void **bvhs, size_t *bvh_bytes);
int  crgpu_scene_create_prepared(const crgpu_prepared *p, int device, crgpu_scene **out);

/* Device memory released by crgpu_scene_destroy is kept in a per-device cache for the next scene (a frame's 35 GB of
 * wavefront state costs 10-55 ms to cudaMalloc and 0.3-0.5 s to cudaFree); crgpu_device_trim returns it to the driver. */
int crgpu_device_trim(int device);
/* Page-locked host memory for buffers that cross PCIe every frame (renderBuffer, scene.c:200); NULL on failure. */
void *crgpu_host_alloc(size_t bytes);
void  crgpu_host_free(void *p);

/* Limit on paths in flight per wavefront batch (default: what fits in 40% of the free device memory at
 * 137 B per path, at most 256M); a tile's passes are processed in batches of floor(max_paths / tile_pixels)
 * passes.  Results do not depend on it; throughput does (every batch pays a fixed latency chain). */
int crgpu_set_max_paths_in_flight(crgpu_scene *s, uint64_t max_paths);

/* Render passes [pass_begin, pass_begin+pass_count) of the tile [x0,x1) x [y0,y1) (y up, end
 * exclusive: `struct renderTile`, tile.h:28-37) into the device framebuffer, continuing the running
 * average stored there.  maxPasses and bounces come from the scene prefs (they seed the sampler,
 * sampler.c:42).  Synchronous (returns when the device is done, `stats` = this call) unless
 * CRGPU_FLAG_ASYNC is given.  `stats` may be NULL.  A tile with more pixels than the paths-in-flight budget
 * is walked in pieces internally. */
int crgpu_render_tile(crgpu_scene *s, int x0, int y0, int x1, int y1,
					  int pass_begin, int pass_count, unsigned flags, struct crgpu_stats *stats);

/* Same, over a UNION of tiles in one wavefront (rects = 4 ints per tile: x0, y0, x1, y1).  This is how a
 * rank of a multi-GPU job renders its share of the tile grid without paying the per-tile launch tails. */
int crgpu_render_tiles(crgpu_scene *s, const int *rects, int nrects,
					   int pass_begin, int pass_count, unsigned flags, struct crgpu_stats *stats);

/* Stopping a render at a pass boundary: renderThread's renderAborted / paused contract (reference renderer.c:258-327).
 * On an ARMED scene every render call checks a stop word in pinned host memory after K1 and before every bounce, and adds each
 * batch of passes to the framebuffer only in pass order and only if no stop was seen during it.  So after any call the
 * framebuffer holds exactly the passes [pass_begin, passes_done) on top of what was there, and a later call for
 * [passes_done, end) finishes the frame bit for bit.  A stop is seen by the next gate, i.e. after the bounce in flight (a pixel set larger than the
 * paths in flight: after the pass batch in flight over the whole set); the call then returns once the batches already queued have
 * drained: each still runs K1 and its bounce launches, on zero rays.  DESIGN §4 has measured latencies (11-49 ms on an H100 at
 * 1-10 s frames).
 *   crgpu_stop_enable   arm (1) or disarm (0); waits for the scene's queued work; arming clears the stop and the progress.
 *                       An unarmed scene renders exactly as before (no gate, no extra kernel).
 *   crgpu_request_stop  one store to pinned memory: thread-safe and async-signal-safe.  It stays set until crgpu_clear_stop, so
 *                       a call made while it is set commits nothing and leaves the framebuffer untouched.
 *   crgpu_progress      no synchronisation: the committed pass index (absolute, starting at pass_begin) of the call in flight
 *                       or of the last one, and whether a call is in flight.
 * A synchronous armed call returns CRGPU_STOPPED when it ended before pass_begin + pass_count; an asynchronous one
 * (CRGPU_FLAG_ASYNC) is read with crgpu_progress.  stats.paths counts the committed passes only.  request_stop, clear_stop and
 * progress on an unarmed scene fail with CRGPU_ERR_BAD_ARGUMENT. */
int crgpu_stop_enable(crgpu_scene *s, int on);
int crgpu_request_stop(crgpu_scene *s);
int crgpu_clear_stop(crgpu_scene *s);
int crgpu_progress(crgpu_scene *s, int *passes_done, int *busy);

/* Reading the image of an armed scene while a call renders it (crGetCurrentImage, reference src/c-ray.h:97).  After each publish
 * step the framebuffer holds exactly the passes [pass_begin, k), so an image taken there is exact: byte for byte the sRGB8 image of
 * a render of [pass_begin, k) on top of what the framebuffer held before the call.  Pixels outside the call's tiles are whatever
 * the framebuffer held.  A pixel set walked in pieces publishes after a pass batch over all of it, so the image always shows one
 * pass boundary over the whole set.
 *   crgpu_request_snapshot  one compare-and-swap on pinned memory: thread-safe and async-signal-safe.  The next publish step
 *                           converts the whole framebuffer to sRGB8 (crgpu_framebuffer_to_srgb8's arithmetic and layout) into a
 *                           device staging buffer of W*H*3 bytes and marks it staged.  A staged image that has not been taken
 *                           stays staged, also past the end of the call: the device never writes the staging buffer until
 *                           crgpu_take_snapshot has copied it, and the pass index it returns says which passes the image shows.
 *   crgpu_take_snapshot     never waits for the render.  With an image staged it copies it to host_rgb8 (W*H*3 bytes) on a stream
 *                           of its own and sets *passes_done (may be NULL) to the pass index it shows.  Otherwise, while a call is
 *                           in flight, it returns CRGPU_PENDING; with no call in flight it converts the framebuffer as it is (on
 *                           the scene's stream, as crgpu_framebuffer_to_srgb8 does) and gives the committed pass index.  Either
 *                           answer completes the request.
 * A render call that finds no request launches the same kernels as before; its publish step stays one thread's work.  Both calls
 * fail with CRGPU_ERR_BAD_ARGUMENT on a NULL or unarmed scene, take also on a NULL buffer; crgpu_stop_enable clears the state. */
int crgpu_request_snapshot(crgpu_scene *s);
int crgpu_take_snapshot(crgpu_scene *s, uint8_t *host_rgb8, int *passes_done);

/* Editing a resident scene between renders (c-ray's crMoveCamera / crTransformMesh, src/c-ray.h:95-103): the edited scene renders
 * the same bits as the scene loaded fresh from the edited JSON.  Both calls first wait for the work queued on the scene's streams,
 * never touch the framebuffer (clear it before rendering the edited frame) and leave the scene unchanged when they fail.
 *   crgpu_scene_set_camera     copies every field of `cam` bit for bit; its width and height must be the scene's image size.
 *   crgpu_scene_set_instances  takes A and Ainv of each instance bit for bit (Ainv is not recomputed); `count`, and each instance's
 *                              kind and object, must be those uploaded (instances cannot be added or removed).  The instance
 *                              boxes, ray offsets and the top-level BVH are rebuilt on the device, the tree that the scene loader
 *                              builds.  The first call gives the scene its own copy of the BVH pair nodes (the uploaded pairs plus
 *                              room for any top level of `count` instances); later calls reuse it.
 * Edits apply to this device scene only: the crgpu_prepared it was created from, and any scene created from that later, are
 * unedited. */
int crgpu_scene_set_camera(crgpu_scene *s, const struct crs_camera *cam);
int crgpu_scene_set_instances(crgpu_scene *s, const struct crs_instance *inst, uint32_t count);

/* Run on a caller-owned CUDA stream (a `cudaStream_t` passed as void*; NULL means the legacy default
 * stream, as everywhere in CUDA).  Lets a host that already has a stream (e.g. the one its NCCL collectives
 * use) order the kernels with its own work and time them with its own events.  crgpu_use_own_stream goes
 * back to the scene's private non-blocking stream. */
int crgpu_set_stream(crgpu_scene *s, void *cuda_stream);
int crgpu_use_own_stream(crgpu_scene *s);
/* Synchronise the stream and return the statistics accumulated since the previous fetch (by
 * crgpu_get_stats or by a synchronous crgpu_render_tile). */
int crgpu_get_stats(crgpu_scene *s, struct crgpu_stats *stats);

/* Framebuffer access.  Host variants copy rows of the tile rectangle (or the whole frame when
 * x1<=x0) between the device framebuffer and a host buffer with the SAME W*H*3 layout. */
int crgpu_framebuffer_clear(crgpu_scene *s);
int crgpu_framebuffer_read(crgpu_scene *s, float *host_rgb, int x0, int y0, int x1, int y1);
int crgpu_framebuffer_write(crgpu_scene *s, const float *host_rgb, int x0, int y0, int x1, int y1);
/* 8-bit sRGB image of the current framebuffer (renderer.c:297-300), W*H*3 bytes, same row order. */
int crgpu_framebuffer_to_srgb8(crgpu_scene *s, uint8_t *host_rgb8);
/* Raw device pointer of the fp32 framebuffer (for the NCCL gather done by the multi-GPU host). */
int crgpu_framebuffer_device_ptr(crgpu_scene *s, void **dev_ptr, size_t *bytes);
/* Device ordinal and image size of a scene (any pointer may be NULL). */
int crgpu_scene_info(crgpu_scene *s, int *device, int *width, int *height);

/* Known-answer hook used by the parity tests: camera ray → closest hit → bsdf sample for `count`
 * (x, y, pass) triples, in the 160-byte record layout of oracle/ref_harness.c `struct hit_kat`. */
int crgpu_trace_kat(crgpu_scene *s, const int32_t *xyp, int count, void *records_out);

/* Test entry point of the traversal kernel that renders frames: closest hits of `n` rays (rays: n x 6 floats, origin then
 * direction) through K2 (k_trace, launched as a frame launches it) and K4 (the counting sort by shading key).  Returns per ray
 * its record, `perm_out` (n ray indices in K4's bucket order: the misses first), `*misses_out` (the number of misses) and in
 * `stats_out` the rays and, with `count`, P/T/S/I.  Fails when the traversal watchdog fired.  Staging of the top BVH nodes
 * follows CRGPU_TRACE_STAGE at crgpu_prepare time and engages for batches of at least 65,536 rays, as in a frame. */
struct crgpu_trace_opts {
	int32_t count;             /* 1: the instrumented kernel, which fills P/T/S/I (it is always built for 3 blocks per SM) */
	int32_t minb;              /* blocks per SM: 2, 3 or 4 */
	int32_t defer;             /* leaf triangles: 0 = in the node step, 1 = after the node burst, 2 = dealt over the warp */
	int32_t refill;            /* a warp fetches rays when fewer than this many lanes are busy: 1..32 */
	int32_t burst;             /* child-pair steps per node phase: >= 1 */
	int32_t inst_min;          /* lanes that must want an instance step before the warp takes one: 1..32 */
	const uint32_t *order;     /* NULL, or a permutation of [0, n): the order K2 takes the rays in (the direction-sorted read) */
};
struct crgpu_ray_record {
	float t, u, v;             /* distance (FLT_MAX for a miss), barycentric u, v of the winning triangle */
	int32_t inst;              /* instance index, -1 = miss */
	int32_t poly;              /* global poly index; -1 for spheres and misses */
	uint32_t key;              /* shading key: 0 for a miss, else min(material + 1, 255) */
	uint32_t prim;             /* triangle slot */
	uint32_t pad;
};
int crgpu_trace_rays(crgpu_scene *s, const float *rays, uint32_t n, const struct crgpu_trace_opts *opts,
                     struct crgpu_ray_record *records_out, uint32_t *perm_out, uint32_t *misses_out, struct crgpu_stats *stats_out);

/* Test entry point of the shading step that renders frames: one bounce of `n` path states through the kernels and launch functions
 * of a frame's bounce — K2 (trace, the frame's trace knobs), K4 (bucket sort), K3 (shade + compaction, in the variant `opts` names)
 * and K4b (direction sort, when `dirmode` is set and depth + 1 < max_depth) — or through the tail kernel, which runs every path to
 * its end (and does nothing when more than 16,384 paths are given).  State i is loaded as path id i with its L; the other half of
 * the wave buffers is poisoned.  Returns per state: K2's record (tail: inst = poly = -2), whether the path continues and its next
 * state (found by the id it was compacted with), L (the L buffer after the step; for a live path meaningful only with has_l),
 * its slot and K3's direction key; `perm2_out` receives K4b's order of the survivors, `*survivors_out` the live count the step left
 * (tail: the live count of the current half) and `box_out` (12 values, may be NULL) dir mode 4's origin-box slot of this depth
 * as it was before the step. */
struct crgpu_path_state {          /* 64 bytes, the layout of struct cro_path_state (oracle/cray_oracle.h) */
	float o[3], d[3];
	float weight[3];
	uint32_t has_l;                /* CRG_ID_HAS_L: L holds radiance */
	uint64_t rng;                  /* PCG state */
	float L[3];
	uint32_t pad;
};
struct crgpu_shade_opts {
	int32_t minb;                  /* K3 hit kernel blocks per SM: 2, 3 or 4 */
	int32_t split;                 /* 1: separate miss kernel */
	int32_t prefetch;              /* 1: perm read ahead + L2 prefetch */
	int32_t dirmode;               /* 0..4: the direction sort of the next bounce (CRGPU_TRACE_SORT) */
	int32_t complete_interpreter;  /* 1: the complete node interpreter even when the scene does not need it */
	int32_t tail;                  /* 1: the tail kernel instead of K2 -> K4 -> K3 */
	int32_t depth, max_depth;      /* the bounce and the scene's bounce limit */
	int32_t generic_only;          /* 1: every hit through the node interpreter; 0: hits on flat materials through the flat launch
	                                  (when split; it then runs at `minb` too) */
};
struct crgpu_shade_result {
	struct crgpu_ray_record rec;
	int32_t alive;
	uint32_t slot;                 /* compacted index of a live path, else 0xffffffff */
	uint32_t dir_key;              /* K3's direction key of a live path (dirmode != 0), else 0xffffffff */
	uint32_t pad;
	struct crgpu_path_state next;
};
int crgpu_shade_rays(crgpu_scene *s, const struct crgpu_path_state *states, uint32_t n, const struct crgpu_shade_opts *opts,
                     struct crgpu_shade_result *results, uint32_t *perm2_out, uint32_t *survivors_out, uint32_t *box_out);

/* The fp64 libm stand-ins of the shading kernels (crgpu_math.cuh) one by one on device `device`: out[i] = f(x[i]) or f(x[i], y[i]). */
enum { CRGPU_LIBM_SIN, CRGPU_LIBM_COS, CRGPU_LIBM_TAN, CRGPU_LIBM_LOG, CRGPU_LIBM_LOG10, CRGPU_LIBM_ATAN2, CRGPU_LIBM_ACOS,
       CRGPU_LIBM_ASIN, CRGPU_LIBM_POW, CRGPU_LIBM_POW5, CRGPU_LIBM_SINCOS_SIN, CRGPU_LIBM_SINCOS_COS, CRGPU_LIBM_COUNT };
int crgpu_libm_eval(int device, int fn, const float *x, const float *y, float *out, uint32_t n);

/* SURVEY §8(f1): the reference's binned-SAH BVH build (reference src/accelerators/bvh.c:96-296: partitionPrimitives,
 * buildBvhRecursive, buildBvhGeneric) on device `device`, level-synchronous (c-ray_b200/csrc/crgpu_bvh_build.cu).  Produces the
 * SAME tree as the reference and as the host builder (crloader_build_bvh): node order, leaf ranges, primitive order, bounds.
 *   bboxes   n x 6 floats: min.x min.y min.z max.x max.y max.z of every primitive (what getBBoxAndCenter returns, bvh.c:283-291)
 *   centers  n x 3 floats
 *   nodes_out  room for 2n-1 nodes;  prims_out  n indices (primIndices);  *node_count_out  nodes written
 * n == 0 writes nothing (an empty BVH, bvh.c:251).  At most 4,194,304 primitives per call. */
int crgpu_bvh_build(const float *bboxes, const float *centers, uint32_t n, int device,
                    struct crs_bvh_node *nodes_out, uint32_t *node_count_out, int32_t *prims_out);

#ifdef __cplusplus
}
#endif
