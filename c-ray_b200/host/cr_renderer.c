/*
 * cr_renderer.c — renderFrame and the GPU worker thread.
 *
 * renderFrame restates reference src/renderer/renderer.c:40-180: allocate the 8-bit output, start
 * prefs.threadCount workers through the thread-function slot, poll their renderThreadState every 16 ms
 * (progress line ~4x/s: percentage of tiles, μs/path, ETA, Msamples/s — renderer.c:126-158), join, return the
 * image.  The workers are gpuRenderThread (one per CUDA device) instead of renderThread (renderer.c:258-327):
 * same tile array, same published fields, same pause flag, but a worker takes its whole share of the tiles at once (a spatial
 * interleave, see gpuRenderThread) and hands it to crgpu_render_tiles as ONE wavefront; pixels never touch the CPU.
 *
 * Per frame a worker uploads the prepared scene (one pinned host->device copy, in parallel on all GPUs), renders,
 * and releases its replica into libcrgpu's per-device cache.  With more than one GPU the tiles are gathered on
 * device 0 / rank 0 by one NCCL exchange (include/crgpu_nccl.h) over a communicator that outlives the frame.
 */
#include "cr_host.h"
#include "../../include/crgpu_nccl.h"
#include <dlfcn.h>
#include "../../include/crloader.h"
#include <strings.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <math.h>
#include <time.h>

/* The NCCL tile gather lives in its own library (libcrgpu_nccl.so) and is loaded on first use: a single-GPU render never
 * touches NCCL, and a host process that already carries an NCCL build (e.g. a Python launcher with torch) binds to the one
 * already mapped (same soname) instead of getting a second.  Looked up next to this library, then on the default search path. */
static struct {
	void *lib;
	int (*create)(const int *, int, crgpu_comm **);
	int (*gather)(crgpu_comm *, crgpu_scene **, const int *, const int *, int, int);
	int (*unique_id)(void *);
	int (*create_rank)(const void *, int, int, int, crgpu_comm **);
	int (*gather_rank)(crgpu_comm *, crgpu_scene *, const int *, const int *, int, int);
	int (*destroy)(crgpu_comm *);
} g_nccl;

int crhost_load_nccl(void) {
	if (g_nccl.gather) return 0;
	char path[4096] = "";
	Dl_info info;
	if (dladdr((void *)crhost_load_nccl, &info) && info.dli_fname) {
		const char *slash = strrchr(info.dli_fname, '/');
		if (slash) snprintf(path, sizeof path, "%.*s/libcrgpu_nccl.so", (int)(slash - info.dli_fname), info.dli_fname);
	}
	void *lib = path[0] ? dlopen(path, RTLD_NOW | RTLD_LOCAL) : NULL;
	if (!lib) lib = dlopen("libcrgpu_nccl.so", RTLD_NOW | RTLD_LOCAL);
	if (!lib) { fprintf(stderr, "renderFrame: cannot load libcrgpu_nccl.so: %s\n", dlerror()); return -1; }
	g_nccl.create = (int (*)(const int *, int, crgpu_comm **))dlsym(lib, "crgpu_comm_create");
	g_nccl.destroy = (int (*)(crgpu_comm *))dlsym(lib, "crgpu_comm_destroy");
	g_nccl.unique_id = (int (*)(void *))dlsym(lib, "crgpu_comm_unique_id");
	g_nccl.create_rank = (int (*)(const void *, int, int, int, crgpu_comm **))dlsym(lib, "crgpu_comm_create_rank");
	g_nccl.gather_rank = (int (*)(crgpu_comm *, crgpu_scene *, const int *, const int *, int, int))dlsym(lib, "crgpu_comm_gather_tiles_rank");
	void *gather = dlsym(lib, "crgpu_comm_gather_tiles");
	if (!g_nccl.create || !g_nccl.destroy || !gather || !g_nccl.unique_id || !g_nccl.create_rank || !g_nccl.gather_rank) {
		fprintf(stderr, "renderFrame: libcrgpu_nccl.so lacks the crgpu_comm_* entry points\n"); dlclose(lib); return -1;
	}
	g_nccl.lib = lib;
	g_nccl.gather = (int (*)(crgpu_comm *, crgpu_scene **, const int *, const int *, int, int))gather;
	return 0;
}

static double now_s(void) {
	struct timespec ts;
	clock_gettime(CLOCK_MONOTONIC, &ts);
	return ts.tv_sec + 1e-9 * ts.tv_nsec;
}
static void sleep_ms(int ms) { struct timespec ts = { ms / 1000, (long)(ms % 1000) * 1000000L }; nanosleep(&ts, NULL); }

struct renderer *newRenderer(void) {                              /* renderer.c:329-343 */
	struct renderer *r = calloc(1, sizeof *r);
	if (!r) return NULL;
	pthread_mutex_init(&r->state.tileMutex, NULL);
	pthread_mutex_init(&r->state.doneMutex, NULL);
	pthread_mutex_init(&r->state.previewMutex, NULL);
	pthread_cond_init(&r->state.doneCond, NULL);
	r->prefs.threadCount = 1;
	r->prefs.imgType = png;
	r->prefs.imgFilePath = "./";
	r->prefs.imgFileName = "rendered";
	r->world = 1;
	return r;
}

/* ---- SURVEY 8(f1): the loader's BVH builds on the device ------------------------------------------------------------------------ */
static int g_bvh_device;
static int gpu_bvh_builder(const float *bb, const float *ct, uint32_t n, struct crs_bvh_node *nodes, uint32_t *count, int32_t *prims) {
	const int rc = crgpu_bvh_build(bb, ct, n, g_bvh_device, nodes, count, prims);
	if (rc != CRGPU_OK) fprintf(stderr, "cray_b200: device BVH build failed (%s); building on the host\n", crgpu_last_error());
	return rc;
}
void crhostUseGpuBvh(int on, int device, unsigned min_prims) {
	g_bvh_device = device;
	crloader_set_bvh_builder(on ? gpu_bvh_builder : NULL, min_prims);
}
static void gpu_bvh_from_env(void) {
	static int done;
	if (done) return;
	done = 1;
	const char *e = getenv("CRAY_GPU_BVH");
	if (e && *e) crhostUseGpuBvh(1, 0, (unsigned)strtoul(e, NULL, 10));
}

int crhostSetAdaptive(struct renderer *r, int on, float threshold) {
	if (!r || (on && !(isfinite(threshold) && threshold >= 0.f))) return -1;
	r->adaptive = on != 0;
	r->adaptiveThreshold = threshold;
	return 0;
}
const uint32_t *crhostAdaptivePasses(const struct renderer *r) { return r ? r->adaptivePasses : NULL; }

static void drop_prepared(struct renderer *r) { if (r->prepared) { crgpu_prepared_free(r->prepared); r->prepared = NULL; } }

int loadSceneFile(struct renderer *r, const char *path, int width, int height, int samples, int bounces) {
	size_t n = strlen(path);
	gpu_bvh_from_env();
	drop_prepared(r);
	if (n > 5 && !strcasecmp(path + n - 5, ".json")) {
		/* a c-ray JSON scene: parse + build both BVH levels on the host (libcrloader.so, include/crloader.h) */
		if (crloader_load_json(&r->scene, path) != 0) {
			fprintf(stderr, "cray_b200: %s\n", crloader_last_error());
			return -1;
		}
	} else if (crscene_load(&r->scene, path) != 0) return -1;
	return applySceneConfig(r, width, height, samples, bounces);
}

int loadSceneBuf(struct renderer *r, const char *json, const char *assetPath, struct crloader_output *output,
				 int width, int height, int samples, int bounces) {
	gpu_bvh_from_env();
	drop_prepared(r);
	if (crloader_load_json_buf(&r->scene, json, assetPath, output) != 0) {
		fprintf(stderr, "cray_b200: %s\n", crloader_last_error());
		return -1;
	}
	return applySceneConfig(r, width, height, samples, bounces);
}

static void free_render_buffer(struct renderer *r) {
	if (!r->state.renderBuffer) return;
	if (r->renderBufferPinned) crgpu_host_free(r->state.renderBuffer); else free(r->state.renderBuffer);
	r->state.renderBuffer = NULL;
}

/* the preview follows the image size: a blank W*H*3 image whenever the size changes (previewMutex held) */
static void preview_resize_locked(struct renderer *r, size_t bytes) {
	if (r->state.previewBytes == bytes) return;
	free(r->state.preview);
	r->state.preview = calloc(bytes ? bytes : 1, 1);
	r->state.previewBytes = r->state.preview ? bytes : 0;
	for (int t = 0; t < r->state.threadStateCount; ++t) r->state.threadStates[t].previewPasses = 0;
}

int applySceneConfig(struct renderer *r, int width, int height, int samples, int bounces) {
	/* the part of loadScene (src/datatypes/scene.c:111-213) that follows parsing + BVH build */
	crscene_set_config(&r->scene, width, height, samples, bounces);
	r->prefs.imageWidth = r->scene.prefs.image_width;
	r->prefs.imageHeight = r->scene.prefs.image_height;
	r->prefs.sampleCount = (int)r->scene.prefs.sample_count;
	r->prefs.bounces = (int)r->scene.prefs.bounces;
	if (!r->prefs.tileWidth) r->prefs.tileWidth = r->scene.prefs.tile_width ? r->scene.prefs.tile_width : 64;
	if (!r->prefs.tileHeight) r->prefs.tileHeight = r->scene.prefs.tile_height ? r->scene.prefs.tile_height : 64;
	r->prefs.tileOrder = (enum renderOrder)r->scene.prefs.tile_order;
	free(r->state.renderTiles);
	r->state.tileCount = (int)quantizeImage(&r->state.renderTiles, r->prefs.imageWidth, r->prefs.imageHeight,
											r->prefs.tileWidth, r->prefs.tileHeight, r->prefs.tileOrder);   /* scene.c:187-192 */
	free(r->state.tileOwner);
	r->state.tileOwner = calloc((size_t)r->state.tileCount + 1, sizeof(int));
	free_render_buffer(r);
	pthread_mutex_lock(&r->state.previewMutex);
	preview_resize_locked(r, (size_t)r->prefs.imageWidth * r->prefs.imageHeight * 3u);
	pthread_mutex_unlock(&r->state.previewMutex);
	/* renderBuffer (scene.c:200): page-locked when a CUDA device is there, so the frame read-back is one DMA */
	const size_t bytes = (size_t)r->prefs.imageWidth * r->prefs.imageHeight * 3 * sizeof(float);
	r->state.renderBuffer = crgpu_host_alloc(bytes);
	r->renderBufferPinned = r->state.renderBuffer != NULL;
	if (!r->state.renderBuffer) r->state.renderBuffer = malloc(bytes);
	if (r->state.renderBuffer) memset(r->state.renderBuffer, 0, bytes);
	if (r->prepared && crgpu_prepared_update_config(r->prepared, &r->scene) != CRGPU_OK) drop_prepared(r);
	return r->state.renderBuffer && r->state.renderTiles ? 0 : -1;
}

/* ---- GPU group set-up (outside the frame) ------------------------------------------------------------------------------------- */
static void drop_comm(struct renderer *r) {
	if (r->comm && g_nccl.destroy) g_nccl.destroy((crgpu_comm *)r->comm);
	r->comm = NULL; r->commMembers = 0;
}

int prepareGpus(struct renderer *r) {
	if (!r->prepared && crgpu_prepare(&r->scene, &r->prepared) != CRGPU_OK) {
		fprintf(stderr, "prepareGpus: %s\n", crgpu_last_error());
		return -1;
	}
	const int n = r->prefs.threadCount < 1 ? 1 : r->prefs.threadCount;
	if (r->world > 1 || n == 1) return 0;
	if (r->comm && r->commMembers == n) return 0;
	drop_comm(r);
	if (crhost_load_nccl() != 0) return -1;
	int devs[64];
	if (n > 64) return -1;
	for (int i = 0; i < n; ++i) devs[i] = i;
	crgpu_comm *c = NULL;
	if (g_nccl.create(devs, n, &c) != CRGPU_OK) return -1;
	r->comm = c; r->commMembers = n;
	return 0;
}

int crhostUniqueId(void *id128) { return crhost_load_nccl() == 0 && g_nccl.unique_id(id128) == CRGPU_OK ? 0 : -1; }

int joinRanks(struct renderer *r, const void *id128, int rank, int world, int device) {
	if (world < 1 || rank < 0 || rank >= world) return -1;
	drop_comm(r);
	r->rank = rank; r->world = world; r->device = device;
	r->prefs.threadCount = 1;
	if (world == 1) return 0;
	if (crhost_load_nccl() != 0) return -1;
	crgpu_comm *c = NULL;
	if (g_nccl.create_rank(id128, rank, world, device, &c) != CRGPU_OK) return -1;
	r->comm = c; r->commMembers = world;
	return 0;
}

/* One-process-per-GPU jobs: drain the tile queue, keep the tiles of this rank.  Static placement (SURVEY 8e: deterministic, so every
 * rank knows every tile's owner for the gather without talking), interleaved IN SPACE: tile (tx, ty) of the tile grid belongs to
 * rank (tx + 5 ty) % world.  Dealing by queue position (k % world) looks equivalent but is not: the default "fromMiddle" order
 * alternates left and right of the image centre, so with two ranks one of them gets every tile left of the centre — measured with
 * the oracle on hdr.json 1920x1080: 11.6% more rays on the odd positions (max/mean 1.12 for 2, 4 and 8 ranks) against 1.00-1.02 for
 * the spatial interleave (the busiest rank sets the frame time).
 * Fills rects (4 ints per tile) and nums (queue positions); returns the count. */
static int tile_rank(const struct renderer *r, const struct renderTile *t, int world) {
	const unsigned tw = r->prefs.tileWidth ? r->prefs.tileWidth : 1u, th = r->prefs.tileHeight ? r->prefs.tileHeight : 1u;
	return (int)((((unsigned)t->begin.x / tw) + 5u * ((unsigned)t->begin.y / th)) % (unsigned)world);
}
void crhostTileOwners(struct renderer *r, int world, int *owners) {
	if (!r || !owners || world < 1) return;
	for (int i = 0; i < r->state.tileCount; ++i) owners[i] = tile_rank(r, &r->state.renderTiles[i], world);
}
int takeRankTiles(struct renderer *r, int *rects, int *nums) {
	int got = 0;
	const int world = r->world > 1 ? r->world : 1;
	for (;;) {
		struct renderTile tile = nextTile(r);
		if (tile.tileNum == -1) break;
		const int owner = tile_rank(r, &tile, world);
		r->state.tileOwner[tile.tileNum] = owner;
		if (owner != r->rank) continue;
		rects[4 * got] = tile.begin.x; rects[4 * got + 1] = tile.begin.y; rects[4 * got + 2] = tile.end.x; rects[4 * got + 3] = tile.end.y;
		nums[got++] = tile.tileNum;
	}
	return got;
}

/* copy the rows of a worker's tiles from a W*H*3 snapshot into the preview; both have the framebuffer's row order (row H-1-y) */
static void preview_tiles(struct renderer *r, struct renderThreadState *ts, const uint8_t *snap, const int *rects, int got, int passes) {
	const size_t W = r->prefs.imageWidth, H = r->prefs.imageHeight;
	pthread_mutex_lock(&r->state.previewMutex);
	if (r->state.preview && r->state.previewBytes == W * H * 3u) {
		for (int i = 0; i < got; ++i) {
			const int *t = rects + 4 * i;
			for (int y = t[1]; y < t[3]; ++y) {
				const size_t off = ((H - 1u - (size_t)y) * W + (size_t)t[0]) * 3u;
				memcpy(r->state.preview + off, snap + off, (size_t)(t[2] - t[0]) * 3u);
			}
		}
		ts->previewPasses = passes;
	}
	pthread_mutex_unlock(&r->state.previewMutex);
}

void *gpuRenderThread(void *arg) {
	struct renderThreadState *ts = arg;
	struct renderer *r = ts->renderer;
	const bool ranked = r->world > 1;
	const int cap = r->state.tileCount > 0 ? r->state.tileCount : 1;
	int *rects = malloc(sizeof(int) * 4 * (size_t)cap);
	int *nums = malloc(sizeof(int) * (size_t)cap);
	/* this worker's scene replica: one pinned host->device copy of the prepared scene, concurrently on every GPU */
	const int device = ranked ? r->device : ts->thread_num;
	if (!rects || !nums || crgpu_scene_create_prepared(r->prepared, device, &ts->gpu) != CRGPU_OK) {
		fprintf(stderr, "gpuRenderThread[%d]: scene upload to device %d failed: %s\n", ts->thread_num, device, crgpu_last_error());
		ts->error = CRGPU_ERR_CUDA;
		r->state.renderAborted = true;
	}
	while (!ts->error && r->state.isRendering && !r->state.renderAborted) {
		while ((ts->paused || r->state.paused) && !r->state.renderAborted) sleep_ms(16);   /* renderer.c:310-312 */
		int got = 0;
		if (ranked) {
			got = takeRankTiles(r, rects, nums);
		} else {
			/* In-process workers share the reference's tile array but not its one-tile-at-a-time queue (nextTile, tile.c:22-45): a GPU
			 * wants its whole share as ONE wavefront (every trip pays the ~7 ms bounce chain and a tail nothing overlaps), and a share
			 * made of consecutive queue positions is a spatial cluster ("fromMiddle": the centre, where the statue is).  So worker t
			 * takes, once, the tiles the spatial interleave gives it — the same placement as ranks (tile_rank), rather than trips of
			 * queue-consecutive tiles, which left the workers unbalanced. */
			const int workers = r->prefs.threadCount > 0 ? r->prefs.threadCount : 1;
			for (int i = 0; i < r->state.tileCount; ++i) {
				struct renderTile *t = &r->state.renderTiles[i];
				if (tile_rank(r, t, workers) != ts->thread_num) continue;
				rects[4 * got] = t->begin.x; rects[4 * got + 1] = t->begin.y; rects[4 * got + 2] = t->end.x; rects[4 * got + 3] = t->end.y;
				nums[got++] = i;
				t->isRendering = true;
			}
			pthread_mutex_lock(&r->state.tileMutex);
			r->state.finishedTileCount += got;                                     /* what the progress line reads */
			pthread_mutex_unlock(&r->state.tileMutex);
		}
		if (got == 0) break;
		ts->currentTileNum = nums[0];
		ts->tiles = got;
		/* The share is ONE armed, asynchronous call (adaptive: one per round).  Like renderThread's loop (renderer.c:271-320), this thread
		 * polls about every 16 ms: it publishes the committed passes, forwards renderAborted and the pause flags as a stop (the call ends at
		 * the next pass boundary), waits while paused, and resumes from the committed pass: the frame is the same bit for bit. */
		const int spp = r->prefs.sampleCount;
		const double t0 = now_s();
		int rc = crgpu_stop_enable(ts->gpu, 1);
		/* adaptive rounds: the pixels of the share start from a fresh record, and each round's select picks the pixels to render */
		const struct crgpu_adaptive rule = { spp < 16 ? (spp < 2 ? 2u : (uint32_t)spp) : 16u, 16u, (uint32_t)spp, r->adaptiveThreshold, 0.01f };
		uint64_t share_pixels = 0, paths_done = 0;
		for (int i = 0; i < got; ++i) share_pixels += (uint64_t)(rects[4 * i + 2] - rects[4 * i]) * (uint64_t)(rects[4 * i + 3] - rects[4 * i + 1]);
		if (rc == CRGPU_OK && r->adaptive) rc = crgpu_adaptive_reset(ts->gpu);
		bool finished = false;
		int begin = 0;
		/* The live preview: like renderThread, which writes each pixel's running average into the 8-bit image after every pass
		 * (renderer.c:294-300), but at most every CR_PREVIEW_INTERVAL_MS.  The worker asks for a snapshot when its committed pass has
		 * advanced; the device stages it at its next publish step, and this loop copies its tiles out once it is there. */
		const size_t snap_bytes = (size_t)r->prefs.imageWidth * r->prefs.imageHeight * 3u;
		uint8_t *snap = crgpu_host_alloc(snap_bytes);
		const bool snap_pinned = snap != NULL;
		if (!snap) snap = malloc(snap_bytes);
		if (!snap) rc = CRGPU_ERR_NOMEM;
		int shown = 0;
		bool asked = false;
		double last_snap = t0;
		while (rc == CRGPU_OK) {
			int from = begin;
			uint32_t active = 0;
			if (r->adaptive) {
				int to = 0;
				rc = crgpu_adaptive_round(ts->gpu, rects, got, &rule, CRGPU_FLAG_ASYNC, NULL, &active, &from, &to);
				if (rc == CRGPU_OK && active == 0) { finished = true; break; }
			} else {
				if (begin >= spp) { finished = true; break; }
				rc = crgpu_render_tiles(ts->gpu, rects, got, begin, spp - begin, CRGPU_FLAG_ASYNC, NULL);
			}
			if (rc != CRGPU_OK) break;
			int done = from, busy = 1;
			bool stopping = false;
			for (;;) {
				crgpu_progress(ts->gpu, &done, &busy);
				ts->completedSamples = done;
				/* tile-passes done, renderer.c:307; adaptive: the pixel-passes committed, in tiles of the share's mean size */
				ts->totalSamples = r->adaptive ? (paths_done + (uint64_t)(done - from) * active) * (uint64_t)got / (share_pixels ? share_pixels : 1u)
				                               : (uint64_t)done * (uint64_t)got;
				if (ts->totalSamples > 0) ts->avgSampleTime = (long)(1e6 * (now_s() - t0) / (double)ts->totalSamples);
				if (asked || !busy) {
					/* with the call over, take answers from the framebuffer: a stop or pause shows its committed passes at once (a
					 * finished share needs no snapshot: renderFrame's image follows) */
					int k = 0;
					const int trc = asked || (done > shown && done < spp) ? crgpu_take_snapshot(ts->gpu, snap, &k) : CRGPU_PENDING;
					if (trc == CRGPU_OK) { preview_tiles(r, ts, snap, rects, got, k); shown = k; asked = false; last_snap = now_s(); }
					else if (trc != CRGPU_PENDING) {            /* stop the call and wait for it before leaving */
						rc = trc;
						crgpu_request_stop(ts->gpu);
						crgpu_get_stats(ts->gpu, NULL);
						break;
					}
				}
				if (!busy) break;
				if (!asked && done > shown && now_s() - last_snap >= 1e-3 * CR_PREVIEW_INTERVAL_MS) { crgpu_request_snapshot(ts->gpu); asked = true; }
				if (!stopping && (r->state.renderAborted || ts->paused || r->state.paused)) { crgpu_request_stop(ts->gpu); stopping = true; }
				sleep_ms(1);      /* a poll is a few loads of pinned memory; a 16 ms period would add 8 ms to the frame on average */
			}
			if (rc != CRGPU_OK) break;
			struct crgpu_stats st;
			rc = crgpu_get_stats(ts->gpu, &st);
			if (rc != CRGPU_OK) break;
			ts->rays += st.rays;
			paths_done += st.paths;
			begin = done;
			if (!r->adaptive && begin >= spp) { finished = true; break; }
			while ((ts->paused || r->state.paused) && !r->state.renderAborted) sleep_ms(16);   /* renderer.c:310-312 */
			if (r->state.renderAborted) break;
			rc = crgpu_clear_stop(ts->gpu);
		}
		if (snap_pinned) crgpu_host_free(snap); else free(snap);
		if (rc != CRGPU_OK) {
			fprintf(stderr, "gpuRenderThread[%d]: %s\n", ts->thread_num, crgpu_last_error());
			ts->error = rc;
			r->state.renderAborted = true;
			break;
		}
		for (int i = 0; i < got; ++i) {
			r->state.renderTiles[nums[i]].isRendering = false;                    /* renderer.c:315-316 */
			r->state.renderTiles[nums[i]].renderComplete = finished;
		}
		ts->currentTileNum = -1;
		break;                                                                    /* the worker's whole share was one trip */
	}
	free(rects); free(nums);
	pthread_mutex_lock(&r->state.doneMutex);
	ts->threadComplete = true;                                    /* renderer.c:323 */
	ts->currentTileNum = -1;
	pthread_cond_broadcast(&r->state.doneCond);
	pthread_mutex_unlock(&r->state.doneMutex);
	return NULL;
}

/* the pass counts of an adaptive frame: each tile's from the worker that rendered it (a rank: its own tiles only) */
static int collect_passes(struct renderer *r, int n, bool ranked) {
	const size_t W = r->prefs.imageWidth, H = r->prefs.imageHeight;
	free(r->adaptivePasses);
	r->adaptivePasses = calloc(W * H, sizeof(uint32_t));
	uint32_t *mine = malloc(W * H * sizeof(uint32_t));
	int err = r->adaptivePasses && mine ? 0 : CRGPU_ERR_NOMEM;
	for (int t = 0; !err && t < n; ++t) {
		const int who = ranked ? r->rank : t;
		if (crgpu_adaptive_read(r->state.threadStates[t].gpu, mine, NULL) != CRGPU_OK) { err = CRGPU_ERR_CUDA; break; }
		for (int i = 0; i < r->state.tileCount; ++i) {
			const struct renderTile *tl = &r->state.renderTiles[i];
			if (r->state.tileOwner[i] != who) continue;
			for (int y = tl->begin.y; y < tl->end.y; ++y) {
				const size_t off = (H - 1u - (size_t)y) * W + (size_t)tl->begin.x;
				memcpy(r->adaptivePasses + off, mine + off, (size_t)(tl->end.x - tl->begin.x) * sizeof(uint32_t));
			}
		}
	}
	free(mine);
	return err;
}

static double floor_div(double a, double b) { return (double)(long long)(a / b); }
static void smart_time(double sec, char *buf, size_t n) {         /* timer.c smartTime */
	if (sec < 1.0) snprintf(buf, n, "%.0fms", 1e3 * sec);
	else if (sec < 60.0) snprintf(buf, n, "%.0fs", sec);
	else if (sec < 3600.0) snprintf(buf, n, "%.0fm %02.0fs", floor_div(sec, 60.0), sec - 60.0 * floor_div(sec, 60.0));
	else snprintf(buf, n, "%.0fh %02.0fm", floor_div(sec, 3600.0), floor_div(sec - 3600.0 * floor_div(sec, 3600.0), 60.0));
}

struct texture8 *renderFrame(struct renderer *r) {
	const int n = r->prefs.threadCount < 1 ? 1 : r->prefs.threadCount;
	const unsigned W = r->prefs.imageWidth, H = r->prefs.imageHeight;
	const bool ranked = r->world > 1;
	int ndev = 0;
	if (crgpu_device_count(&ndev) != CRGPU_OK || ndev < (ranked ? r->device + 1 : n)) {
		fprintf(stderr, "renderFrame: %d GPU worker(s) requested, %d CUDA device(s) present: %s\n", n, ndev, crgpu_last_error());
		return NULL;
	}
	if (prepareGpus(r) != 0) { fprintf(stderr, "renderFrame: GPU set-up failed\n"); return NULL; }   /* no-op when the host did it already */
	if (ranked && !r->comm) { fprintf(stderr, "renderFrame: rank %d of %d has not joined its group (joinRanks)\n", r->rank, r->world); return NULL; }
	struct texture8 *output = calloc(1, sizeof *output);          /* renderer.c:41 */
	output->width = W; output->height = H;
	output->data = calloc((size_t)W * H * 3, 1);
	pthread_mutex_lock(&r->state.previewMutex);                   /* the preview starts blank, like the output */
	preview_resize_locked(r, (size_t)W * H * 3);
	if (r->state.preview) memset(r->state.preview, 0, r->state.previewBytes);
	pthread_mutex_unlock(&r->state.previewMutex);
	if (r->state.threadStateCount != n) {
		/* a host thread may be reading the worker states (crhostProgress): swap the array under doneMutex, and only when its size
		 * changes; between frames of the same size the entries are re-initialised in place */
		struct renderThreadState *states = calloc((size_t)n, sizeof *states);
		pthread_mutex_lock(&r->state.doneMutex);
		free(r->state.threadStates);
		r->state.threadStates = states;
		r->state.threadStateCount = n;
		pthread_mutex_unlock(&r->state.doneMutex);
	}
	free(r->state.threads);
	r->state.threads = calloc((size_t)n, sizeof *r->state.threads);
	/* every tile's owner (worker or rank) is fixed by the spatial interleave before any worker starts, so that the gather sees the
	 * same table on every rank even when a rank is aborted before it has taken its tiles */
	for (int i = 0; i < r->state.tileCount; ++i) r->state.tileOwner[i] = tile_rank(r, &r->state.renderTiles[i], ranked ? r->world : n);
	bool *started = calloc((size_t)n, sizeof *started);
	r->state.saveImage = true;                                    /* ui.c */
	r->state.renderAborted = false;
	r->state.isRendering = true;
	r->state.finishedTileCount = 0;
	r->state.activeThreads = 0;
	for (int i = 0; i < r->state.tileCount; ++i) { r->state.renderTiles[i].renderComplete = false; r->state.renderTiles[i].isRendering = false; }
	if (!r->prefs.quiet) printf("Rendering %ux%u, %d samples, %d bounces on %d GPU%s, %d tiles\n", W, H, r->prefs.sampleCount,
								r->prefs.bounces, ranked ? r->world : n, (ranked ? r->world : n) > 1 ? "s" : "", r->state.tileCount);
	const double t0 = now_s();
	for (int t = 0; t < n; ++t) {                                 /* renderer.c:97-105 */
		r->state.threadStates[t] = (struct renderThreadState){ .thread_num = t, .renderer = r, .currentTileNum = -1 };
		if (pthread_create(&r->state.threads[t], NULL, gpuRenderThread, &r->state.threadStates[t]) == 0) { started[t] = true; r->state.activeThreads++; }
		else {                                                    /* renderer.c:100-101 logs and carries on with the threads it has */
			fprintf(stderr, "renderFrame: failed to create a render thread\n");
			r->state.threadStates[t].threadComplete = true;
			r->state.threadStates[t].error = CRGPU_ERR_CUDA;
		}
	}
	int pauser = 0;
	while (r->state.isRendering) {                                /* renderer.c:122-172 */
		{	/* renderer.c:171 sleeps 16 ms (active_msec) between polls; here a finishing worker ends the wait early */
			struct timespec until;
			clock_gettime(CLOCK_REALTIME, &until);
			const long add_ns = (r->state.threadStates[0].paused ? 100L : 16L) * 1000000L;
			until.tv_nsec += add_ns;
			if (until.tv_nsec >= 1000000000L) { until.tv_sec += 1; until.tv_nsec -= 1000000000L; }
			pthread_mutex_lock(&r->state.doneMutex);
			int alldone = 1;
			for (int t = 0; t < n; ++t) alldone &= r->state.threadStates[t].threadComplete ? 1 : 0;
			if (!alldone) pthread_cond_timedwait(&r->state.doneCond, &r->state.doneMutex, &until);
			pthread_mutex_unlock(&r->state.doneMutex);
		}
		if (!r->prefs.quiet && ++pauser >= 280 / 16) {            /* the progress line, ~4x/s (renderer.c:137-158) */
			pauser = 0;
			uint64_t done = 0, mine = 0;
			for (int t = 0; t < n; ++t) { done += r->state.threadStates[t].totalSamples; mine += (uint64_t)r->state.threadStates[t].tiles; }
			/* this process' share of the tile-passes: the whole frame in-process, this rank's tiles in a ranked job */
			const uint64_t all = (mine ? mine : (uint64_t)r->state.tileCount) * (uint64_t)r->prefs.sampleCount;
			const double el = now_s() - t0;
			const double usPerPath = done ? 1e6 * el / ((double)done * r->prefs.tileWidth * r->prefs.tileHeight) : 0.0;
			char rem[64];
			smart_time(done ? el * (double)(all - done) / (double)done : 0.0, rem, sizeof rem);
			printf("[%.0f%%] us/path: %.04f, etf: %s, %.02lfMs/s %s        \r", 100.0 * (double)done / (double)(all ? all : 1),
				   usPerPath, done ? rem : "?", usPerPath > 0.0 ? 1.0 / usPerPath : 0.0,
				   r->state.threadStates[0].paused || r->state.paused ? "[PAUSED]" : "");
			fflush(stdout);
		}
		int done = 0;
		for (int t = 0; t < n; ++t) done += r->state.threadStates[t].threadComplete ? 1 : 0;
		if (done == n) r->state.isRendering = false;
	}
	for (int t = 0; t < n; ++t) if (started[t]) pthread_join(r->state.threads[t], NULL);   /* renderer.c:175-177 */
	free(started);
	r->state.activeThreads = 0;
	int err = 0;
	r->state.totalRays = 0;
	for (int t = 0; t < n; ++t) { err |= r->state.threadStates[t].error; r->state.totalRays += r->state.threadStates[t].rays; }
	crgpu_scene *root_scene = r->state.threadStates[0].gpu;
	const bool discard = !err && r->state.renderAborted && !r->state.saveImage;   /* aborted without saving (ui.c) */

	/* a rank takes part in the gather even when it discards its frame: every rank of the group must enter the collective */
	if (!err && (ranked || (n > 1 && !discard))) {
		/* every tile's owner is known (state.tileOwner): gather the float tiles on device 0 / rank 0 */
		int *rects = malloc(sizeof(int) * 4 * (size_t)r->state.tileCount);
		for (int i = 0; i < r->state.tileCount; ++i) {
			const struct renderTile *t = &r->state.renderTiles[i];
			rects[4 * i] = t->begin.x; rects[4 * i + 1] = t->begin.y; rects[4 * i + 2] = t->end.x; rects[4 * i + 3] = t->end.y;
		}
		if (ranked) {
			if (g_nccl.gather_rank((crgpu_comm *)r->comm, root_scene, rects, r->state.tileOwner, r->state.tileCount, 0) != CRGPU_OK) err = CRGPU_ERR_CUDA;
		} else {
			crgpu_scene **scenes = calloc((size_t)n, sizeof *scenes);
			for (int t = 0; t < n; ++t) scenes[t] = r->state.threadStates[t].gpu;
			if (g_nccl.gather((crgpu_comm *)r->comm, scenes, rects, r->state.tileOwner, r->state.tileCount, 0) != CRGPU_OK) err = CRGPU_ERR_CUDA;
			free(scenes);
		}
		free(rects);
	}
	if (!err && !discard && (!ranked || r->rank == 0)) {
		if (crgpu_framebuffer_read(root_scene, r->state.renderBuffer, 0, 0, 0, 0) != CRGPU_OK) err = CRGPU_ERR_CUDA;   /* renderBuffer, scene.c:200 */
		if (!err && crgpu_framebuffer_to_srgb8(root_scene, output->data) != CRGPU_OK) err = CRGPU_ERR_CUDA;            /* renderer.c:297-300 */
	}
	r->state.renderSeconds = now_s() - t0;
	if (!err && r->adaptive) err = collect_passes(r, n, ranked);
	for (int t = 0; t < n; ++t) if (r->state.threadStates[t].gpu) { crgpu_scene_destroy(r->state.threadStates[t].gpu); r->state.threadStates[t].gpu = NULL; }
	if (!r->prefs.quiet && !err && !discard) {
		const double samples = (double)W * H * r->prefs.sampleCount;
		printf("\nFinished render in %.3f s: %.2f Msample/s, %.2f Mray/s (%llu rays)\n", r->state.renderSeconds,
			   samples / r->state.renderSeconds / 1e6, (double)r->state.totalRays / r->state.renderSeconds / 1e6, (unsigned long long)r->state.totalRays);
	}
	if (discard && !r->prefs.quiet) printf("\nAborted: image not saved\n");
	if (err || discard) { destroyTexture8(output); return NULL; }
	if (!ranked || r->rank == 0) {                                /* the preview ends on the frame's image */
		pthread_mutex_lock(&r->state.previewMutex);
		if (r->state.preview && r->state.previewBytes == (size_t)W * H * 3) memcpy(r->state.preview, output->data, r->state.previewBytes);
		for (int t = 0; t < n; ++t) r->state.threadStates[t].previewPasses = r->state.threadStates[t].completedSamples;
		pthread_mutex_unlock(&r->state.previewMutex);
	}
	return output;
}

void crhostAbort(struct renderer *r, int save) {
	if (!r) return;
	r->state.saveImage = save != 0;
	r->state.renderAborted = true;
}
void crhostSetPaused(struct renderer *r, int on) { if (r) r->state.paused = on != 0; }
/* the worker states are read under doneMutex: renderFrame swaps the array under it when the worker count changes */
int crhostProgress(const struct renderer *r, unsigned long long *passes_done_total) {
	if (!r) return 0;
	unsigned long long done = 0;
	pthread_mutex_t *m = (pthread_mutex_t *)&r->state.doneMutex;
	pthread_mutex_lock(m);
	for (int t = 0; t < r->state.threadStateCount; ++t) done += r->state.threadStates[t].totalSamples;
	pthread_mutex_unlock(m);
	if (passes_done_total) *passes_done_total = done;
	return r->state.isRendering ? 1 : 0;
}
int crhostCurrentImagePasses(struct renderer *r, uint8_t *rgb8, int *passes, int workers) {
	if (!r) return 0;
	pthread_mutex_lock(&r->state.doneMutex);                      /* the worker states (see crhostProgress), then the preview */
	pthread_mutex_lock(&r->state.previewMutex);
	/* exactly the W*H*3 bytes of the current image size, whatever the preview holds */
	const size_t bytes = (size_t)r->prefs.imageWidth * r->prefs.imageHeight * 3u;
	if (rgb8 && r->state.preview && r->state.previewBytes == bytes) memcpy(rgb8, r->state.preview, bytes);
	else if (rgb8) memset(rgb8, 0, bytes);
	for (int t = 0; passes && t < workers && t < r->state.threadStateCount; ++t) passes[t] = r->state.threadStates[t].previewPasses;
	pthread_mutex_unlock(&r->state.previewMutex);
	pthread_mutex_unlock(&r->state.doneMutex);
	return r->state.isRendering ? 1 : 0;
}
int crhostCurrentImage(struct renderer *r, uint8_t *rgb8) { return crhostCurrentImagePasses(r, rgb8, NULL, 0); }
int crhostWorkerPasses(const struct renderer *r, int t) {
	if (!r) return 0;
	pthread_mutex_t *m = (pthread_mutex_t *)&r->state.doneMutex;
	pthread_mutex_lock(m);
	const int passes = t >= 0 && t < r->state.threadStateCount ? r->state.threadStates[t].completedSamples : 0;
	pthread_mutex_unlock(m);
	return passes;
}

void destroyTexture8(struct texture8 *t) { if (t) { free(t->data); free(t); } }

void destroyRenderer(struct renderer *r) {                       /* renderer.c:346-362 */
	if (!r) return;
	drop_comm(r);
	drop_prepared(r);
	crscene_free(&r->scene);
	free_render_buffer(r);
	free(r->state.renderTiles); free(r->state.tileOwner); free(r->state.threads); free(r->state.threadStates);
	free(r->state.preview);
	free(r->adaptivePasses);
	pthread_mutex_destroy(&r->state.previewMutex);
	pthread_mutex_destroy(&r->state.tileMutex);
	pthread_mutex_destroy(&r->state.doneMutex);
	pthread_cond_destroy(&r->state.doneCond);
	free(r);
}

/* ---- small accessors for hosts that bind libcrhost.so through an FFI and do not want to mirror struct layouts ------------------- */
float *crhostRenderBuffer(struct renderer *r) { return r ? r->state.renderBuffer : NULL; }
double crhostRenderSeconds(const struct renderer *r) { return r ? r->state.renderSeconds : 0.0; }
unsigned long long crhostTotalRays(const struct renderer *r) { return r ? (unsigned long long)r->state.totalRays : 0ull; }
void crhostConfigure(struct renderer *r, int gpus, unsigned tileWidth, unsigned tileHeight, int quiet) {
	if (!r) return;
	if (gpus > 0) r->prefs.threadCount = gpus;
	if (tileWidth) r->prefs.tileWidth = tileWidth;
	if (tileHeight) r->prefs.tileHeight = tileHeight;
	r->prefs.quiet = quiet != 0;
}
void crhostImageSize(const struct renderer *r, unsigned *w, unsigned *h, int *samples, int *bounces) {
	if (!r) return;
	if (w) *w = r->prefs.imageWidth;
	if (h) *h = r->prefs.imageHeight;
	if (samples) *samples = r->prefs.sampleCount;
	if (bounces) *bounces = r->prefs.bounces;
}

void *crhostComm(struct renderer *r) { return r ? r->comm : NULL; }
const void *crhostPrepared(struct renderer *r) { return r ? r->prepared : NULL; }
int crhostTileCount(const struct renderer *r) { return r ? r->state.tileCount : 0; }
/* rank/world of a job WITHOUT joining an NCCL group (tile-assignment logic only; used by CPU tests and by hosts that gather themselves) */
void crhostSetRank(struct renderer *r, int rank, int world) { if (r && world >= 1 && rank >= 0 && rank < world) { r->rank = rank; r->world = world; } }
void crhostResetQueue(struct renderer *r) { if (r) { pthread_mutex_lock(&r->state.tileMutex); r->state.finishedTileCount = 0; pthread_mutex_unlock(&r->state.tileMutex); } }
