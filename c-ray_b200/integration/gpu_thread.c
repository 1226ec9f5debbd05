/*
 * gpu_thread.c — REFERENCE-SIDE integration code (INTEGRATION.md §2): the worker a c-ray maintainer adds as
 * src/renderer/gpu_thread.c.  It occupies the thread-function slot of `struct crThread` that renderFrame fills with
 * renderThread (reference src/renderer/renderer.c:92-105, src/utils/platform/thread.h:22-31) and calls ONLY the C ABI of
 * include/crgpu.h.  Compiles against the reference's headers; built by oracle/Makefile (`cray_ref_gpu`) together with the
 * unmodified reference sources, never into libcrgpu.so / libcrhost.so.
 *
 * Differences from renderThread (renderer.c:258-327), all inside this worker:
 *   - the scene is flattened once per process (flatten_world) and uploaded to the worker's device (thread_num = CUDA device);
 *   - a trip to the tile queue takes several tiles (a GPU wavefront wants ~64M paths in flight; one 64x64 tile is 4096 pixels)
 *     and renders them as ONE wavefront with crgpu_render_tiles;
 *   - pixels land in the device framebuffer and are copied into state.renderBuffer / the 8-bit output per tile afterwards, with
 *     the layout of setPixel (texture.c:19-28), so the preview window, the stats loop and the encoders see what they expect;
 *   - while a trip renders, the 8-bit output of its tiles is refreshed from snapshots (crgpu_request_snapshot /
 *     crgpu_take_snapshot) at most every GPU_PREVIEW_INTERVAL_MS, so the preview improves during the trip as renderThread's
 *     does pass by pass (renderer.c:294-300).  The float renderBuffer is written once, at the end of the trip.
 */
#include "includes.h"
#include "renderer/renderer.h"
#include "datatypes/tile.h"
#include "datatypes/scene.h"
#include "datatypes/image/texture.h"
#include "utils/platform/thread.h"
#include "utils/platform/mutex.h"
#include "utils/logging.h"
#include "utils/timer.h"

#include <stdlib.h>
#include <string.h>
#include <pthread.h>

#include "crgpu.h"

int flatten_world(const struct renderer *r, struct crs_scene *out);

static pthread_mutex_t g_flat_lock = PTHREAD_MUTEX_INITIALIZER;
static struct crs_scene g_flat;
static crgpu_prepared *g_prepared;
static const struct world *g_flat_of;

/* flatten + re-layout once per loaded scene; every GPU worker then uploads the same prepared scene */
static crgpu_prepared *prepared_scene(const struct renderer *r) {
	pthread_mutex_lock(&g_flat_lock);
	if (g_flat_of != r->scene || !g_prepared) {
		if (g_prepared) { crgpu_prepared_free(g_prepared); g_prepared = NULL; }
		if (flatten_world(r, &g_flat) == 0 && crgpu_prepare(&g_flat, &g_prepared) == 0) g_flat_of = r->scene;
		else g_prepared = NULL;
	} else {
		/* same world, possibly other prefs (-d / -s between frames): header only */
		g_flat.prefs.image_width = r->prefs.imageWidth; g_flat.prefs.image_height = r->prefs.imageHeight;
		g_flat.prefs.sample_count = (uint32_t)r->prefs.sampleCount; g_flat.prefs.bounces = (uint32_t)r->prefs.bounces;
		crgpu_prepared_update_config(g_prepared, &g_flat);
	}
	crgpu_prepared *p = g_prepared;
	pthread_mutex_unlock(&g_flat_lock);
	return p;
}

#define GPU_TRIP_MAX 1024
#define GPU_PREVIEW_INTERVAL_MS 100      /* the host mirror's CR_PREVIEW_INTERVAL_MS */

/* the rows of a trip's tiles from a W*H*3 image in setPixel's layout (texture.c:24-28) into another */
static void copy_tile_rows(unsigned char *dst, const unsigned char *src, const int *rects, int got, unsigned W, unsigned H) {
	for (int i = 0; i < got; ++i) {
		const int *q = rects + 4 * i;
		for (int y = q[1]; y < q[3]; ++y) {
			const size_t off = ((size_t)q[0] + (size_t)(H - (unsigned)(y + 1)) * W) * 3u;
			memcpy(dst + off, src + off, (size_t)(q[2] - q[0]) * 3u);
		}
	}
}

void *gpuRenderThread(void *arg) {
	struct renderThreadState *ts = (struct renderThreadState *)threadUserData(arg);      /* thread.c:15-18 */
	struct renderer *r = ts->renderer;
	struct texture *image = ts->output;
	crgpu_scene *gpu = NULL;
	crgpu_prepared *prepared = prepared_scene(r);
	if (!prepared || crgpu_scene_create_prepared(prepared, ts->thread_num /* = CUDA device */, &gpu) != CRGPU_OK) {
		logr(warning, "GPU worker %i: %s\n", ts->thread_num, crgpu_last_error());
		ts->threadComplete = true;
		ts->currentTileNum = -1;
		return 0;
	}
	const unsigned W = r->prefs.imageWidth, H = r->prefs.imageHeight;
	const double tilePaths = (double)r->prefs.tileWidth * r->prefs.tileHeight * (double)r->prefs.sampleCount;
	int *rects = malloc(sizeof(int) * 4 * GPU_TRIP_MAX);
	int *nums = malloc(sizeof(int) * GPU_TRIP_MAX);
	float *fb = malloc(sizeof(float) * 3 * (size_t)W * H);          /* same W*H*3 layout as renderBuffer; only tile rectangles are touched */
	unsigned char *fb8 = malloc((size_t)3 * W * H);
	struct timeval timer = {0};
	ts->completedSamples = 1;
	while (r->state.isRendering) {
		int want = (int)(64.0 * 1048576.0 / (tilePaths > 1.0 ? tilePaths : 1.0)) + 1;
		const int left = r->state.tileCount - r->state.finishedTileCount;
		const int share = (left + r->prefs.threadCount - 1) / (r->prefs.threadCount > 0 ? r->prefs.threadCount : 1);
		if (want > share) want = share;
		if (want > GPU_TRIP_MAX) want = GPU_TRIP_MAX;
		if (want < 1) want = 1;
		int got = 0;
		while (got < want) {
			struct renderTile tile = nextTile(r);                                        /* tile.c:22-45 */
			if (tile.tileNum == -1) break;
			rects[4 * got] = tile.begin.x; rects[4 * got + 1] = tile.begin.y; rects[4 * got + 2] = tile.end.x; rects[4 * got + 3] = tile.end.y;
			nums[got++] = tile.tileNum;
		}
		if (got == 0) break;
		ts->currentTileNum = nums[0];
		startTimer(&timer);
		/* One armed, asynchronous call per trip, polled like renderThread checks its flags (renderer.c:271-320): renderAborted and
		 * paused become a stop at a pass boundary (after the bounce in flight and the drain of the queued batches, DESIGN §4);
		 * while paused the worker waits, then resumes from the committed pass, which leaves the tiles bit-identical to an
		 * uninterrupted trip. */
		const uint64_t samplesBefore = ts->totalSamples;
		int begin = 0, rc = crgpu_stop_enable(gpu, 1);
		int shown = 0, asked = 0;
		long lastSnapUs = 0;
		while (rc == CRGPU_OK && begin < r->prefs.sampleCount) {
			rc = crgpu_render_tiles(gpu, rects, got, begin, r->prefs.sampleCount - begin, CRGPU_FLAG_ASYNC, NULL);
			int done = begin, busy = rc == CRGPU_OK, stopping = 0;
			while (busy) {
				crgpu_progress(gpu, &done, &busy);
				/* what the stats loop of renderFrame reads (renderer.c:126-158) */
				ts->completedSamples = done > 0 ? done : 1;
				ts->totalSamples = samplesBefore + (uint64_t)done * (uint64_t)got;
				if (done > 0) ts->avgSampleTime = getUs(timer) / ((long)done * got);
				if (asked) {                 /* staged by a publish step; or, once the call is over, the framebuffer as it is */
					int k = 0;
					if (crgpu_take_snapshot(gpu, fb8, &k) == CRGPU_OK) {
						copy_tile_rows(image->data.byte_p, fb8, rects, got, W, H);
						shown = k; asked = 0; lastSnapUs = getUs(timer);
					}
				}
				if (busy && !asked && done > shown && getUs(timer) - lastSnapUs >= 1000L * GPU_PREVIEW_INTERVAL_MS) { crgpu_request_snapshot(gpu); asked = 1; }
				if (!stopping && (r->state.renderAborted || ts->paused)) { crgpu_request_stop(gpu); stopping = 1; }
				if (busy) sleepMSec(1);
			}
			if (rc == CRGPU_OK) rc = crgpu_get_stats(gpu, NULL);
			begin = done;
			if (begin >= r->prefs.sampleCount || r->state.renderAborted) break;
			while (ts->paused && !r->state.renderAborted) sleepMSec(16);                   /* renderer.c:310-312 */
			if (rc == CRGPU_OK) rc = crgpu_clear_stop(gpu);
		}
		if (rc != CRGPU_OK) {
			logr(warning, "GPU worker %i: %s\n", ts->thread_num, crgpu_last_error());
			break;
		}
		/* renderer.c:294-300: the float tile into state.renderBuffer, the sRGB tile into the 8-bit output */
		crgpu_framebuffer_to_srgb8(gpu, fb8);
		copy_tile_rows(image->data.byte_p, fb8, rects, got, W, H);
		for (int i = 0; i < got; ++i) {
			const int *q = rects + 4 * i;
			crgpu_framebuffer_read(gpu, fb, q[0], q[1], q[2], q[3]);
			for (int y = q[1]; y < q[3]; ++y) {
				const size_t off = ((size_t)q[0] + (size_t)(H - (unsigned)(y + 1)) * W) * 3u;       /* texture.c:24-28 */
				memcpy(r->state.renderBuffer->data.float_p + off, fb + off, (size_t)(q[2] - q[0]) * 3u * sizeof(float));
			}
			r->state.renderTiles[nums[i]].isRendering = false;                           /* renderer.c:315-316 */
			r->state.renderTiles[nums[i]].renderComplete = begin >= r->prefs.sampleCount;
		}
		ts->currentTileNum = -1;
		ts->completedSamples = 1;
		if (r->state.renderAborted) break;                                                 /* renderer.c:272 */
	}
	free(rects); free(nums); free(fb); free(fb8);
	crgpu_scene_destroy(gpu);
	ts->threadComplete = true;                                                            /* renderer.c:323 */
	ts->currentTileNum = -1;
	return 0;
}
