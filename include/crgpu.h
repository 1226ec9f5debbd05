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

/* Editing a resident scene between renders (c-ray's crMoveCamera / crTransformMesh / crSetHDR, src/c-ray.h:95-103): the edited scene
 * renders the same bits as the scene loaded fresh from the edited JSON.  Every call first waits for the work queued on the scene's streams,
 * never touch the framebuffer (clear it before rendering the edited frame) and leave the scene unchanged when they fail.
 *   crgpu_scene_set_camera     copies every field of `cam` bit for bit; its width and height must be the scene's image size.
 *   crgpu_scene_set_instances  takes A and Ainv of each instance bit for bit (Ainv is not recomputed); `count`, and each instance's
 *                              kind and object, must be those of the scene's current list (crgpu_scene_set_instance_list changes
 *                              them).  The instance boxes, ray offsets and the top-level BVH are rebuilt on the device, the tree that
 *                              the scene loader builds.  The first instance or mesh edit gives the scene its own copy of the BVH pair
 *                              nodes (the uploaded pairs plus room for any top level of `count` instances) and its own top-level item
 *                              records; later edits reuse them.  A top level that needs more than count - 1 pair nodes (a tree of more
 *                              than 2 count - 1 nodes, which only instances whose boxes no split separates make: see
 *                              crloader_build_bvh in crloader.h) or is deeper than 64 levels is refused with CRGPU_ERR_UNSUPPORTED.
 *   crgpu_scene_set_instance_list  replaces the whole instance list: instance i of `inst` becomes instance i of the scene, `count`
 *                              from 0 to 4,194,304 (the device builder's limit; above it CRGPU_ERR_UNSUPPORTED before any instance is
 *                              read).  Each instance is a CRS_INST_SPHERE or CRS_INST_MESH of a sphere or mesh of the scene (uploaded
 *                              or added by crgpu_scene_add_objects), also one that had no instance; this call creates no object.  A
 *                              sphere instance takes its sphere's radius and material, a mesh instance its mesh's current BVH (crgpu_scene_set_meshes included), and every object
 *                              the ray offset of its last instance, as the scene loader gives them.  A and Ainv are taken bit for bit.
 *                              A NULL `inst` with count > 0, another kind or an object out of range is refused with
 *                              CRGPU_ERR_BAD_ARGUMENT; a top level of more than 2 count - 1 nodes or deeper than 64 levels with
 *                              CRGPU_ERR_UNSUPPORTED.  With count 0 every ray misses.  The instance records, instance keys,
 *                              last-instance table and item records then live in an instance block that only grows (the upload's
 *                              instance sections stay allocated, unread); a top level that no longer fits the top region gets a
 *                              larger region at the end of the pairs block, and mesh regions never move.  Later calls of
 *                              crgpu_scene_set_instances and crgpu_scene_set_meshes work on the new list.
 *   crgpu_scene_set_meshes     deforms meshes (crTransformMesh, "recompute kd-tree"): every mesh listed in `meshes` takes its polys,
 *                              flat->polys[poly_offset .. + poly_count), and the vertices, normals and texture coordinates they
 *                              index from `flat`; positions, normals, uvs and each poly's material (within the mesh's material
 *                              range) may change.  Nothing else in `flat` is read: its BVHs and ray offsets are ignored and rebuilt.
 *                              Exactly the listed meshes are rebuilt: a vertex shared with an unlisted mesh does not move that mesh.
 *                              Each listed mesh's record must equal the uploaded one in poly_offset, poly_count, material_offset,
 *                              material_count, texcoord_count and bvh, and its uploaded BVH must cover exactly its polys; a mesh
 *                              out of range, a mesh listed twice, an index out of range or a material outside the mesh's range is
 *                              refused with CRGPU_ERR_BAD_ARGUMENT, as crgpu_prepare refuses them.  On the device, each mesh's
 *                              triangle boxes, BVH (the tree the scene loader builds), leaf-ordered triangles and shading records are
 *                              rebuilt, then every instance's box and ray offset under its current transform (an earlier
 *                              crgpu_scene_set_instances included) and the top level.  A mesh tree of more than 2n - 1 nodes
 *                              (crloader_build_bvh), deeper than 64 levels, or of more than 4,194,304 polys is refused with
 *                              CRGPU_ERR_UNSUPPORTED.  The first edit of a mesh gives it its own region of max(1, n - 1) pair nodes
 *                              behind the scene's other pairs; later edits reuse it.
 *   crgpu_scene_set_shading    replaces the materials, the node graph, the textures, the texel data and the background root
 *                              (crSetHDR, and recolouring, re-bsdf'ing or lighting surfaces) with those of `flat`, reading only its
 *                              material_count, materials, node_count, nodes, texture_count, textures, texdata_bytes, texdata and
 *                              background.  material_count must be the scene's count, as uploaded or as crgpu_scene_add_objects left it (else CRGPU_ERR_BAD_ARGUMENT): material i of
 *                              `flat` becomes material i of the scene, and which material each poly and sphere uses does not change
 *                              (crgpu_scene_set_meshes changes a poly's).  Node count, texture count and texel bytes may grow or
 *                              shrink.  The arrays are validated and folded as crgpu_prepare does it, and a refusal returns the code
 *                              crgpu_prepare returns for them.  Materials, flat records and K4's key order are rewritten in place; the
 *                              nodes, texture table and all texel data are uploaded on every call into a new block that replaces the
 *                              previous edit's (the upload's node and texel sections stay allocated, unread).
 *   crgpu_scene_add_objects    puts new meshes and spheres into the scene (crLoadMeshFromFile): `flat` is the grown scene B as a whole
 *                              (the loader places every mesh's materials before the spheres', so adding a mesh moves every sphere's
 *                              material).  With M meshes, S spheres and P polys in the scene, B's first M meshes and S spheres are the
 *                              scene's: mesh m < M equals the scene's record in poly_offset, poly_count, material_offset,
 *                              material_count, texcoord_count and bvh and keeps its current geometry (B's polys, vertices, normals
 *                              and texcoords for it are not read); sphere s < S keeps its radius bit for bit and takes B's material.
 *                              Each new mesh's polys lie at or above P inside B's poly_count, apart from every other new mesh's; its
 *                              indices and poly materials are checked as crgpu_prepare checks them, its material range lies inside
 *                              B's materials, and its bvh index is below B's bvh_count, is not B's top_bvh and no other mesh's.  From
 *                              the call on B's BVH indices name the scene's BVH records; B's bvhs, bvh_nodes and prim_indices are not
 *                              read: each new mesh's tree (the one the scene loader builds), triangles and shading records are built
 *                              on the device.  New spheres take B's radius and material.  B's materials, nodes, textures, texel data
 *                              and background replace the scene's as crgpu_scene_set_shading takes them, at B's material count, and
 *                              B's instance list replaces the scene's as crgpu_scene_set_instance_list takes it; prefs and camera are
 *                              not read.  When B's first M meshes hold the scene's current geometry the scene then renders, traces and
 *                              shades the bits of B loaded fresh.  A NULL argument, fewer meshes or spheres than the scene holds, a
 *                              changed record, a poly range out of bounds or shared, a bad bvh index, an index or material out of range
 *                              is refused with CRGPU_ERR_BAD_ARGUMENT; a new mesh of more than 4,194,304 polys or a tree deeper than
 *                              64 levels, more than 2^32 triangle slots, or an instance list set_instance_list refuses with
 *                              CRGPU_ERR_UNSUPPORTED; shading is refused with the code crgpu_prepare returns.  The triangles, slot
 *                              records, shading records and BVH records then live in a geometry block that grows by half at least
 *                              when it is outgrown (new meshes take slots and pair regions behind the existing ones, which never
 *                              move), the materials in a materials block replaced when B's count outgrows it; the upload's sections
 *                              stay allocated, unread.  Framebuffers and views are not touched.  Every other edit then works on the
 *                              grown scene.
 *   crgpu_scene_shading        the live scene's counterpart of crgpu_prepared_materials and crgpu_prepared_background (same kinds and
 *                              flags, read back from the device: min(count, material count) entries), and whether the shading kernels
 *                              run the complete node interpreter.  kinds and flags may be NULL when count is 0, the other outputs
 *                              always.
 * Edits apply to this device scene only: the crgpu_prepared it was created from, and any scene created from that later, are
 * unedited. */
int crgpu_scene_set_camera(crgpu_scene *s, const struct crs_camera *cam);
int crgpu_scene_set_instances(crgpu_scene *s, const struct crs_instance *inst, uint32_t count);
int crgpu_scene_set_instance_list(crgpu_scene *s, const struct crs_instance *inst, uint32_t count);
int crgpu_scene_set_meshes(crgpu_scene *s, const struct crs_scene *flat, const uint32_t *meshes, uint32_t count);
int crgpu_scene_set_shading(crgpu_scene *s, const struct crs_scene *flat);
int crgpu_scene_add_objects(crgpu_scene *s, const struct crs_scene *flat);
int crgpu_scene_shading(crgpu_scene *s, uint32_t *kinds, uint32_t *flags, uint32_t count, uint32_t *material_count,
                        uint32_t *background_kind, int *complete_interpreter);

/* Rendering several views of a resident scene in one call (c-ray's scene.h cameraCount, "Currently only one camera supported"): stereo
 * pairs, turntables, camera rigs, thumbnails.  A scene has a list of views, each a camera and a framebuffer of the scene's image size;
 * after upload it has one.  View 0 IS the scene's camera and framebuffer: crgpu_render_tile(s), crgpu_framebuffer_*, snapshots and
 * crgpu_trace_kat work on it as before, and crgpu_scene_set_camera sets its camera.
 *   crgpu_scene_set_views   takes `count` cameras (1 .. CRGPU_MAX_VIEWS) bit for bit, each of the scene's image size; cams[0] becomes the
 *                           scene camera.  Like the edits above it first waits for the queued work and leaves the scene unchanged when it
 *                           fails: a NULL scene or cams, a count of 0 or above the limit, or a camera of another size is refused with
 *                           CRGPU_ERR_BAD_ARGUMENT, a failed allocation with CRGPU_ERR_NOMEM.  It never changes a surviving view's pixels:
 *                           views 0 .. min(old, new count) - 1 keep their framebuffers, views beyond the old count start zeroed.  The
 *                           cameras and framebuffers of views 1 .. count - 1 live in one views block from the per-device cache, which
 *                           only grows and goes back to the cache at crgpu_scene_destroy; the paths-in-flight budget is not changed.
 *   crgpu_render_views      renders passes [pass_begin, pass_begin + pass_count) of the tile set `rects` (as crgpu_render_tiles takes
 *                           it, and sharing its cached device pixel list) in each view [first_view, first_view + view_count) as ONE
 *                           wavefront: one set of batches, and one tail per batch, for all of them.  Afterwards each of those views'
 *                           framebuffers holds, bit for bit, what crgpu_render_tiles(rects, pass_begin, pass_count) gives after
 *                           crgpu_scene_set_camera(its camera) on the same framebuffer contents; other views are untouched.  The views
 *                           share their sampler seeds by design (a seed depends on pixel, pass and sample count only: sampler.c:41-44),
 *                           which is what makes each view equal to its single render; their noise is therefore correlated.  The call
 *                           numbers its (view, pixel) pairs view-major and cuts them into pieces of at most max_paths as one pixel set;
 *                           flags work as in crgpu_render_tiles.  stats.paths is view_count x pixels x passes; rays and, with
 *                           CRGPU_FLAG_COUNT, P/T/S/I are the sums of the views' single renders.  A view range outside the list, more
 *                           than 2^32 - 1 (view, pixel) pairs, or a tile set crgpu_render_tiles refuses is refused (nothing rendered).
 *                           On an armed scene the call is pass-major over all its pairs, so one committed pass index holds for every
 *                           view: crgpu_request_stop ends it at a pass boundary, crgpu_progress reports it, and a later call for
 *                           [committed, end) finishes every view bit for bit.  A views call stages no snapshot: a request made during it
 *                           stays pending (crgpu_take_snapshot returns CRGPU_PENDING while it runs) and is served afterwards as always,
 *                           by the next publishing call or by crgpu_take_snapshot with no call in flight (view 0's framebuffer).
 *   crgpu_scene_view_count  the number of views in the list.
 *   crgpu_view_clear / crgpu_view_read / crgpu_view_to_srgb8
 *                           zero, copy out (W*H*3 floats in the framebuffer layout) or convert to sRGB8 (crgpu_framebuffer_to_srgb8's
 *                           arithmetic and layout, W*H*3 bytes) the whole framebuffer of one view of the list.
 * crgpu_scene_set_instances, _set_instance_list, _set_meshes, _set_shading and _add_objects do not touch the views; every view renders the edited
 * scene. */
#define CRGPU_MAX_VIEWS 65536u
int crgpu_scene_set_views(crgpu_scene *s, const struct crs_camera *cams, uint32_t count);
int crgpu_scene_view_count(crgpu_scene *s, uint32_t *count);
int crgpu_render_views(crgpu_scene *s, uint32_t first_view, uint32_t view_count, const int *rects, int nrects,
                       int pass_begin, int pass_count, unsigned flags, struct crgpu_stats *stats);
int crgpu_view_clear(crgpu_scene *s, uint32_t view);
int crgpu_view_read(crgpu_scene *s, uint32_t view, float *host_rgb);
int crgpu_view_to_srgb8(crgpu_scene *s, uint32_t view, uint8_t *host_rgb8);

/* Changing the render settings of a resident scene between renders (c-ray's crSetImageWidth / crSetImageHeight / crSetSampleCount /
 * crSetBounces, src/c-ray.h:58-74): a viewport resize, a low-sample preview followed by the final render, another bounce limit.
 *   crgpu_scene_set_render  sets the image size, sample count and bounce limit, and the cameras of the view list.  Like the edits above
 *                           it first waits for the work queued on the scene's streams and leaves the scene exactly as it was when it
 *                           fails (framebuffers, views, cameras and snapshot state included).  Afterwards the scene renders, traces and
 *                           shades (crgpu_render_tile(s), crgpu_render_views, crgpu_trace_kat, crgpu_trace_rays, crgpu_shade_rays) the
 *                           bits of a fresh scene of its current content, every earlier edit included, given these four settings and
 *                           these cameras: what crscene_set_config, crgpu_prepare and crgpu_scene_create_prepared would give it.
 *                           width, height and sample_count of 0 are refused with CRGPU_ERR_BAD_ARGUMENT, as crgpu_prepare refuses them;
 *                           every bounce limit crgpu_prepare takes is taken, 0 included (every sample is then black).  `count` must be
 *                           crgpu_scene_view_count and every camera width x height: cams[0] becomes the scene camera and cams[v] the
 *                           camera of view v, taken bit for bit.  cams may be NULL only when width and height are the scene's: every
 *                           camera is then kept.  Any other NULL, another count or a camera of another size is refused with
 *                           CRGPU_ERR_BAD_ARGUMENT; the view list keeps its length (crgpu_scene_set_views changes it).
 *                           With the image size unchanged no framebuffer is touched, as with every other edit.  A new size gives view
 *                           0 and each other view a new framebuffer of that size, zeroed, and the views block room for the current
 *                           view count only.  All new blocks are allocated first (a failure returns CRGPU_ERR_NOMEM and changes
 *                           nothing), the scene is published, and only then the old blocks go back to the per-device cache: a pointer
 *                           crgpu_framebuffer_device_ptr gave before a size change is dead afterwards, so a host that holds one (the
 *                           NCCL gather) asks again.  The sRGB8 staging buffers of crgpu_framebuffer_to_srgb8 and of snapshots go back
 *                           to the cache too and are allocated again at the new size when next used: an image staged before the size
 *                           change is dropped, while a pending request stays pending and is served at the new size.  An armed scene
 *                           stays armed, with its stop word and progress as they were.  The paths-in-flight budget is not changed.
 *                           crgpu_scene_info, every rectangle check, the framebuffer and view accessors and snapshots use the new size;
 *                           a cached tile set is checked against it before it is used again. */
int crgpu_scene_set_render(crgpu_scene *s, uint32_t width, uint32_t height, uint32_t sample_count, uint32_t bounces,
                           const struct crs_camera *cams, uint32_t count);

/* Rendering adaptively (DESIGN §4 "Rendering adaptively"): each pixel stops taking passes once its error estimate falls below a
 * threshold, so flat sky or a diffuse wall far from any caustic stops early while noisy pixels go on to pass_end.  Every pixel of view 0
 * has a record: n, the passes its framebuffer holds; the Welford mean and M2 of their luminance y = (0.2126 r + 0.7152 g) + 0.0722 b;
 * the error of its last test; and a done bit.  Only K5 updates n, mean and M2, and only for the passes it commits.  The test points are
 * k = min_passes + j round_passes below pass_end; at one, err = sqrt(M2 / (n - 1) / n) / max(mean, floor) (fp32), and the pixel is done
 * when err < threshold (a NaN err never stops it).  The decision depends on the pixel's own samples only, and paths are seeded by
 * (pixel, pass, sample count) only, so a pixel that holds n passes holds bit for bit what crgpu_render_tiles(rects, 0, n) gives it on a
 * cleared framebuffer, whatever the tiling, pieces, paths in flight, path order, worker split or stops in between.
 *   crgpu_adaptive_reset  allocates the adaptive block from the per-device cache the first time (16 B of record per pixel, plus the
 *                         active list and the select's scratch: 44 B per pixel in all) and sets every record to n = 0, err = +inf, not
 *                         done.  It waits for the scene's queued work.  crgpu_scene_set_render with a new size drops the block: a round
 *                         is then refused until the next reset.  No other edit touches the records, as edits leave framebuffers alone.
 *                         The block goes back to the cache at crgpu_scene_destroy.
 *   crgpu_adaptive_round  one round over the tile set `rects` (as crgpu_render_tiles takes it, sharing its cached pixel list): a select
 *                         step tests each pixel of the set that is not done and whose n is a test point, then compacts the pixels that
 *                         are not done and have n < pass_end, in list order, into the active list and reads back their number and the
 *                         min and max of their n (the round's one synchronisation).  With min = max = k it renders passes [k, next) of
 *                         the active pixels as crgpu_render_tiles renders a pixel set (pieces, batches, flags, stop gates, progress,
 *                         snapshots), where next is the smallest test point above k, capped at pass_end.  It returns *active, and
 *                         *pass_begin = k, *pass_end_of_round = next; with no active pixel it renders nothing, returns CRGPU_OK and sets
 *                         both to pass_end.  An armed round that is stopped returns CRGPU_STOPPED; the next round resumes from the
 *                         committed pass.  stats as for crgpu_render_tiles (paths: the pixel-passes rendered), kernel_launches including
 *                         the select's.  A NULL scene, a, active, pass_begin or pass_end_of_round, a field of `a` out of range, a
 *                         scene with no adaptive block, a tile list crgpu_render_tiles refuses, tiles that overlap (K5 would add one
 *                         pixel twice at once), and active pixels of different counts (two overlapping tile sets left at different
 *                         passes) are refused with CRGPU_ERR_BAD_ARGUMENT; a refused round changes no record and no framebuffer pixel.
 *                         Rounds work on view 0 only.
 *   crgpu_adaptive_read   waits for the scene's stream and copies n and err of every pixel (W*H each, framebuffer order: row H-1-y
 *                         first); either pointer may be NULL. */
struct crgpu_adaptive {
	uint32_t min_passes;    /* >= 2: the first convergence test is at this pass count */
	uint32_t round_passes;  /* >= 1: later tests every round_passes passes */
	uint32_t pass_end;      /* 1 .. the scene's sample_count: no pixel goes beyond it */
	float    threshold;     /* finite, >= 0: a pixel stops when err < threshold (so 0 never stops a pixel early) */
	float    floor;         /* finite, > 0: the mean luminance below which err is taken relative to `floor` */
};
int crgpu_adaptive_reset(crgpu_scene *s);
int crgpu_adaptive_round(crgpu_scene *s, const int *rects, int nrects, const struct crgpu_adaptive *a, unsigned flags,
                         struct crgpu_stats *stats, uint32_t *active, int *pass_begin, int *pass_end_of_round);
int crgpu_adaptive_read(crgpu_scene *s, uint32_t *passes, float *err);

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
/* Raw device pointer of the fp32 framebuffer (for the NCCL gather done by the multi-GPU host).  A size change by
 * crgpu_scene_set_render replaces the framebuffer: the pointer given before it is dead afterwards. */
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

/* Test entry points of the accumulation kernel (K5) and of an adaptive round's select, scan and compaction, on given samples and
 * records instead of rendered ones (tests/test_gpu_adaptive_kernels.py).
 *   crgpu_accumulate_samples  passes [pass_begin, +pass_count) of the tile set `rects` (as crgpu_render_tiles takes it) from given
 *                         radiance: L holds npix x pass_count x 4 floats, pixel by pixel in the tile set's list order, then pass by
 *                         pass (the fourth float is not read).  Each sample goes to the slot of the wave buffers' radiance that path
 *                         order `order` (0..7, or -1: the process's CRGPU_PATH_ORDER) gives its (pass, pixel), and K5 runs with the
 *                         grid and tile descriptor of an unarmed render call, over the scene's framebuffer; with `adaptive` it runs
 *                         the adaptive instantiation, which also updates the pixels' records (crgpu_adaptive_reset first).
 *                         pixels_out (may be NULL) receives the list: npix words x | y << 16.  Refused with CRGPU_ERR_BAD_ARGUMENT: a
 *                         NULL scene or L, an order out of range, adaptive without records, a tile list crgpu_render_tiles refuses,
 *                         passes outside [0, sample_count), and npix x pass_count above the paths in flight.
 *   crgpu_adaptive_write / crgpu_adaptive_records  load / copy out the whole record of every pixel of view 0 (W*H, framebuffer
 *                         order, as crgpu_adaptive_read).  Each waits for the scene's stream.
 *   crgpu_adaptive_select the select, scan and compaction of crgpu_adaptive_round (the same code, refused in the same cases, with the
 *                         same records left behind) without the render that follows: active_out (room for the tile set's pixels)
 *                         receives the active list, *count_out its length, *lo_out and *hi_out the least and the largest count of
 *                         its pixels (0xffffffff and 0 with none active).  Refused active pixels of different counts name both in the
 *                         error text. */
struct crgpu_adaptive_record {
	uint32_t n;             /* passes taken; bit 31 (CRGPU_ADAPTIVE_DONE): the pixel has converged */
	float    mean, m2;      /* Welford mean and M2 of the luminance of those passes */
	float    err;           /* the error of the last test (+inf before the first) */
};
#define CRGPU_ADAPTIVE_DONE 0x80000000u
int crgpu_accumulate_samples(crgpu_scene *s, const int *rects, int nrects, int pass_begin, int pass_count, int order, int adaptive,
                             const float *L, uint32_t *pixels_out);
int crgpu_adaptive_write(crgpu_scene *s, const struct crgpu_adaptive_record *recs);
int crgpu_adaptive_records(crgpu_scene *s, struct crgpu_adaptive_record *recs_out);
int crgpu_adaptive_select(crgpu_scene *s, const int *rects, int nrects, const struct crgpu_adaptive *a, uint32_t *active_out,
                          uint32_t *count_out, uint32_t *lo_out, uint32_t *hi_out);

/* The path order of the frame path (CRGPU_PATH_ORDER, c-ray_b200/csrc/crgpu_wave.cuh), evaluated on the host for order `order`
 * (0..7): for a batch of npix pixels and pass_count passes, pass_out[id] and pixel_out[id] are the pass and pixel (local to the
 * batch) that path id renders, id_out[pass * npix + pixel] is the path id of that pair (any of the three may be NULL); and, when
 * w and h are not 0, xy_out[i] = x | y << 16 is pixel i of a w x h rectangle in that order's pixel order.  Needs no device. */
int crgpu_path_order_map(int order, uint32_t npix, uint32_t pass_count, uint32_t *pass_out, uint32_t *pixel_out, uint32_t *id_out,
                         uint32_t w, uint32_t h, uint32_t *xy_out);

/* SURVEY §8(f1): the reference's binned-SAH BVH build (reference src/accelerators/bvh.c:96-296: partitionPrimitives,
 * buildBvhRecursive, buildBvhGeneric) on device `device`, level-synchronous (c-ray_b200/csrc/crgpu_bvh_build.cu).  Produces the
 * SAME tree as the reference and as the host builder (crloader_build_bvh): node order, leaf ranges, primitive order, bounds.
 *   bboxes   n x 6 floats: min.x min.y min.z max.x max.y max.z of every primitive (what getBBoxAndCenter returns, bvh.c:283-291)
 *   centers  n x 3 floats
 *   nodes_out  room for 2n-1 nodes;  prims_out  n indices (primIndices);  *node_count_out  nodes written
 * n == 0 writes nothing (an empty BVH, bvh.c:251).  At most 4,194,304 primitives per call.
 * A tree with empty leaves can need more than 2n-1 nodes (see crloader_build_bvh in crloader.h): then nothing is written to nodes_out
 * or prims_out, *node_count_out is set to the number of nodes the tree needs and CRGPU_ERR_UNSUPPORTED is returned. */
int crgpu_bvh_build(const float *bboxes, const float *centers, uint32_t n, int device,
                    struct crs_bvh_node *nodes_out, uint32_t *node_count_out, int32_t *prims_out);

#ifdef __cplusplus
}
#endif
