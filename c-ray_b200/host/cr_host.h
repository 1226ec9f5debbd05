/*
 * cr_host.h — host-side C mirror of c-ray's renderer / tile dispatcher, with GPU worker threads.
 *
 * Same names, argument meaning and division of labour as the reference so that the hot path drops in
 * behind the existing dispatcher:
 *   struct renderTile          reference src/datatypes/tile.h:28-37
 *   quantizeImage / nextTile   reference src/datatypes/tile.c:66-117 / :22-45
 *   struct renderThreadState   reference src/renderer/renderer.h:14-31 (the fields workers publish)
 *   struct renderer / prefs    reference src/renderer/renderer.h:58-98 (the subset this path needs)
 *   renderFrame                reference src/renderer/renderer.c:40-180
 *   gpuRenderThread            occupies the thread-function slot of renderThread (renderer.c:258-327)
 *   writeImage                 reference src/utils/encoders/encoder.c:22-39 (PNG / BMP, 8-bit sRGB)
 *
 * The scene arrives as the flat description of include/crscene.h (what c-ray's loader + BVH builder
 * produce, flattened); everything the workers compute happens in libcrgpu.so (include/crgpu.h).
 * Plain C99 + pthreads.  No CPU rendering path exists here.
 */
#pragma once
#include <stdbool.h>
#include <stdint.h>
#include <pthread.h>
#include "../../include/crgpu.h"
#include "../../include/crloader.h"

struct intCoord { int x, y; };

enum renderOrder {                 /* tile.h:15-21 */
	renderOrderTopToBottom = 0,
	renderOrderFromMiddle,
	renderOrderToMiddle,
	renderOrderNormal,
	renderOrderRandom
};

struct renderTile {                /* tile.h:28-37 */
	unsigned width, height;
	struct intCoord begin, end;    /* end exclusive, y up */
	bool isRendering, renderComplete, networkRenderer;
	int tileNum;
};

enum fileType { bmp = 0, png = 1 };

struct texture8 {                  /* the char_p texture renderFrame returns (renderer.c:41) */
	unsigned width, height;
	uint8_t *data;                 /* W*H*3, row 0 = image top */
};

struct renderer;

struct renderThreadState {         /* renderer.h:14-31 */
	int thread_num;                /* = CUDA device ordinal of this worker */
	bool threadComplete;
	bool paused;                   /* set by the host (reference: the 'p' key, ui.c): the worker stops at a pass boundary until cleared */
	int currentTileNum;
	int completedSamples;
	uint64_t totalSamples;
	long avgSampleTime;            /* microseconds per tile-pass */
	struct renderer *renderer;
	crgpu_scene *gpu;              /* this worker's device-resident scene replica */
	uint64_t rays;                 /* closest-hit queries traced by this worker */
	int error;                     /* first CRGPU_ERR_* seen, 0 = none */
	int tiles;                     /* tiles of this worker's share (the denominator of its progress) */
	int previewPasses;             /* passes its tiles show in state.preview (under previewMutex) */
};

struct prefs {                     /* renderer.h:58-87 */
	enum renderOrder tileOrder;
	int threadCount;               /* = number of GPU workers */
	int sampleCount, bounces;
	unsigned tileWidth, tileHeight;
	unsigned imageWidth, imageHeight;
	const char *imgFilePath, *imgFileName;
	int imgCount;
	enum fileType imgType;
	bool quiet;
};

struct state {                     /* renderer.h:34-55 */
	struct renderTile *renderTiles;
	int tileCount, finishedTileCount;
	int *tileOwner;                /* worker (= device) that rendered each tile, for the multi-GPU gather */
	float *renderBuffer;           /* fp32 W*H*3, row H-1-y (scene.c:200, texture.c:24-28) */
	int activeThreads;
	bool isRendering, renderAborted;
	bool saveImage;                /* ui.c: false when the frame was aborted without saving (renderFrame then returns no image) */
	bool paused;                   /* crhostSetPaused: every worker pauses, as with its own renderThreadState::paused */
	pthread_t *threads;
	struct renderThreadState *threadStates;
	int threadStateCount;          /* entries of threadStates: kept across frames (and swapped under doneMutex) so that
	                                  crhostProgress may read them from any thread */
	pthread_mutex_t tileMutex;
	pthread_mutex_t doneMutex;     /* workers signal doneCond when they finish: renderFrame wakes up at once instead of at its next 16 ms poll */
	pthread_cond_t doneCond;
	double renderSeconds;
	uint64_t totalRays;
	/* the live 8-bit image of the frame (W*H*3, the layout of struct texture8): blank when a frame starts, each worker's tiles
	 * refreshed from GPU snapshots while it renders (gpuRenderThread), the final image once the frame is done */
	uint8_t *preview;
	size_t previewBytes;
	pthread_mutex_t previewMutex;
};

struct renderer {
	struct crs_scene scene;        /* flat scene (owned) */
	struct state state;
	struct prefs prefs;
	crgpu_prepared *prepared;      /* the scene re-laid out for the kernels, pinned host memory (built once per scene, like the
	                                  BVHs of loadScene, scene.c:111-213); every frame uploads it to the worker GPUs */
	/* one-process-per-GPU jobs (torchrun / mpirun style; the counterpart of the reference's cluster workers,
	 * src/utils/protocol/worker.c): this process renders the tiles whose queue position % world == rank on `device` */
	int rank, world, device;
	void *comm;                    /* crgpu_comm*: persistent NCCL communicator (in-process group or this rank's membership) */
	int commMembers;               /* size of the group `comm` was created for */
	bool renderBufferPinned;
};

/* tile dispatcher */
unsigned quantizeImage(struct renderTile **renderTiles, unsigned width, unsigned height,
					   unsigned tileWidth, unsigned tileHeight, enum renderOrder tileOrder);
struct renderTile nextTile(struct renderer *r);

/* renderer */
struct renderer *newRenderer(void);
int loadSceneFile(struct renderer *r, const char *json_or_crscene_path, int width, int height, int samples, int bounces);
int loadSceneBuf(struct renderer *r, const char *json, const char *assetPath, struct crloader_output *output,
				 int width, int height, int samples, int bounces);   /* loadScene(r, buf), scene.c:121 */
/* (re)derive prefs, tile grid and host framebuffer from r->scene after -d/-s style overrides (<= 0 keeps a value) */
int applySceneConfig(struct renderer *r, int width, int height, int samples, int bounces);
struct texture8 *renderFrame(struct renderer *r);          /* NULL on error */
void destroyTexture8(struct texture8 *t);
void destroyRenderer(struct renderer *r);

/* loads libcrgpu_nccl.so (multi-GPU tile gather) on first use; 0 when its entry points are available */
int crhost_load_nccl(void);
/* GPU group set-up, OUTSIDE the frame (NCCL bootstrap takes 0.1-1 s per group, once per process):
 *   prepareGpus     in-process group for renderFrame with prefs.threadCount > 1 (also done lazily by renderFrame)
 *   crhostUniqueId  rank 0 of a multi-process job makes the 128-byte id the launcher distributes
 *   joinRanks       every process of the job: I am `rank` of `world`, rendering on CUDA device `device` */
int prepareGpus(struct renderer *r);
int crhostUniqueId(void *id128);
int joinRanks(struct renderer *r, const void *id128, int rank, int world, int device);

/* accessors for FFI hosts (no struct mirroring needed) */
float *crhostRenderBuffer(struct renderer *r);
double crhostRenderSeconds(const struct renderer *r);
unsigned long long crhostTotalRays(const struct renderer *r);
void crhostConfigure(struct renderer *r, int gpus, unsigned tileWidth, unsigned tileHeight, int quiet);
/* SURVEY 8(f1): build the BVHs of the scenes loaded after this call on CUDA device `device` (crgpu_bvh_build) when they have at
 * least min_prims primitives; on == 0 goes back to the host builder.  Same tree either way.  Also switched on by the environment
 * variable CRAY_GPU_BVH=<min_prims> (read by loadSceneFile / loadSceneBuf). */
void crhostUseGpuBvh(int on, int device, unsigned min_prims);
void crhostImageSize(const struct renderer *r, unsigned *w, unsigned *h, int *samples, int *bounces);
void *crhostComm(struct renderer *r);
const void *crhostPrepared(struct renderer *r);
int crhostTileCount(const struct renderer *r);
void crhostSetRank(struct renderer *r, int rank, int world);
void crhostResetQueue(struct renderer *r);
int takeRankTiles(struct renderer *r, int *rects, int *nums);
void crhostTileOwners(struct renderer *r, int world, int *owners);   /* owner rank of every tile, in queue order */
/* Controls of a frame in flight, for hosts without the reference's UI (ui.c: Ctrl-C / 'X' abort without saving, 'S' aborts and
 * saves, 'P' pauses).  Workers stop at a pass boundary after the bounce in flight and the drain of the batches already queued
 * (crgpu_request_stop; measured latencies in DESIGN §4); after an abort with save,
 * renderFrame returns the committed passes of every worker, after one without it returns no image.
 *   crhostProgress  1 while a frame renders, else 0; *passes_done_total = tile-passes committed by all workers so far
 *   crhostWorkerPasses  the passes worker t has committed (its tiles hold exactly passes [0, that)) */
void crhostAbort(struct renderer *r, int save);
void crhostSetPaused(struct renderer *r, int on);
int crhostProgress(const struct renderer *r, unsigned long long *passes_done_total);
int crhostWorkerPasses(const struct renderer *r, int t);
/* The image of the frame as it stands, from any thread (crGetCurrentImage, reference src/c-ray.h:97): copies W*H*3 bytes into
 * rgb8 and returns 1 while a frame renders, else 0 (the last frame's image, or blank before the first).  While a frame renders,
 * each worker's tiles show the sRGB8 image of exactly the passes [0, k) it had committed at its latest snapshot; a worker takes
 * one when its committed pass has advanced and CR_PREVIEW_INTERVAL_MS has passed since its previous one.  A rank of a
 * one-process-per-GPU job shows its own tiles only, and only rank 0 (which receives the gathered frame) ends on the frame's
 * image: another rank keeps its last snapshot of its own tiles.  The image always has the current image size: after a size
 * change (applySceneConfig) it is blank until the next frame.  crhostCurrentImagePasses also gives, read under the same lock, the pass
 * count k each worker's tiles show (passes[t] for t < min(workers, worker count)). */
#define CR_PREVIEW_INTERVAL_MS 100
int crhostCurrentImage(struct renderer *r, uint8_t *rgb8);
int crhostCurrentImagePasses(struct renderer *r, uint8_t *rgb8, int *passes, int workers);

/* worker entry point with the signature of renderThread (void *(*)(void *)) */
void *gpuRenderThread(void *arg);

/* encoders: 8-bit RGB, rows top to bottom */
int writeImage(const struct texture8 *img, const char *path, enum fileType type);
int encodeBMP(const struct texture8 *img, const char *path);
int encodePNG(const struct texture8 *img, const char *path);
/* what the reference stores in the PNG's tEXt chunks (struct renderInfo, src/datatypes/image/imagefile.h:13-21; png.c:29-56) */
struct renderInfo { int samples, bounces, threadCount; double renderSeconds; };
int encodePNGInfo(const struct texture8 *img, const char *path, const struct renderInfo *info);
int writeImageInfo(const struct texture8 *img, const char *path, enum fileType type, const struct renderInfo *info);
void rendererInfo(const struct renderer *r, struct renderInfo *out);
