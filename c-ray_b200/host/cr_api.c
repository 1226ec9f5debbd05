/*
 * cr_api.c — c-ray's public library API (include/cray_api.h) on top of the host mirror.
 *
 * Mirrors reference src/c-ray.c function by function; the global renderer, the option table filled by crParseArgs
 * (reference src/utils/args.c:70-262) and the "current image" handed from crStartRenderer to crWriteImage are the same
 * three pieces of process state the reference keeps (c-ray.c:28-30, args.c:26).
 */
#ifndef _GNU_SOURCE
#define _GNU_SOURCE
#endif
#include "../../include/cray_api.h"
#include "cr_host.h"
#include <libgen.h>
#include <pthread.h>
#include <stdarg.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

static struct renderer *g_renderer;
static struct texture8 *g_image;
static pthread_mutex_t g_image_lock = PTHREAD_MUTEX_INITIALIZER;   /* crGetCurrentImage may run while crStartRenderer renders */
static char *g_asset_path;
static struct crloader_output g_output;
static bool g_antialiasing = true;

/* ---- options: a small string -> value table (the reference's constantsDatabase, args.c:26) ------------------ */
struct option { char *key; char *str; int num; };
static struct option *g_opts;
static int g_nopts;

static struct option *opt_find(const char *key) {
	for (int i = 0; i < g_nopts; ++i) if (!strcmp(g_opts[i].key, key)) return &g_opts[i];
	return NULL;
}
static struct option *opt_set(const char *key) {
	struct option *o = opt_find(key);
	if (o) return o;
	g_opts = realloc(g_opts, sizeof(*g_opts) * (size_t)(g_nopts + 1));
	g_opts[g_nopts] = (struct option){ strdup(key), NULL, 0 };
	return &g_opts[g_nopts++];
}
static void opt_int(const char *key, int v) { opt_set(key)->num = v; }
static void opt_str(const char *key, const char *v) { struct option *o = opt_set(key); free(o->str); o->str = strdup(v); }
static int opt_get(const char *key) { struct option *o = opt_find(key); return o ? o->num : 0; }

static bool file_ok(const char *p) { FILE *f = fopen(p, "r"); if (f) fclose(f); return f != NULL; }

static bool parse_dims(const char *s, int *w, int *h) {            /* args.c:47-68 */
	if (!s) return false;
	const char *x = strchr(s, 'x');
	int W = atoi(s), H = x ? atoi(x + 1) : 0;
	W = W > 65536 ? 65536 : W; H = H > 65536 ? 65536 : H;
	W = W < 1 ? 1 : W; H = H < 1 ? 1 : H;
	*w = W; *h = H;
	return true;
}

/* ---- version / environment ------------------------------------------------------------------------------------ */
char *crGetVersion(void) { return "0.6.3-b200"; }
char *crGitHash(void) { return "b200path"; }
bool isDebug(void) { return false; }
void crInitialize(void) { setvbuf(stdout, NULL, _IOLBF, 0); }

void crLog(const char *fmt, ...) {
	char buf[512];
	va_list vl;
	va_start(vl, fmt);
	vsnprintf(buf, sizeof(buf), fmt, vl);
	va_end(vl);
	printf("[info] %s", buf);
}

/* ---- command line ------------------------------------------------------------------------------------------------ */
void crParseArgs(int argc, char **argv) {
	bool inputSet = opt_find("inputFile") != NULL;
	for (int i = 1; i < argc; ++i) {
		char *alt = NULL;
		if (asprintf(&alt, "%s.json", argv[i]) < 0) alt = NULL;
		if (!inputSet && file_ok(argv[i])) { opt_str("inputFile", argv[i]); inputSet = true; }
		else if (!inputSet && alt && file_ok(alt)) { opt_str("inputFile", alt); inputSet = true; }
		free(alt);
		const char *next = i + 1 < argc ? argv[i + 1] : NULL;
		if (!strcmp(argv[i], "-h")) {
			printf("Usage: %s [-hjsdt] [input_json...]\n"
				   "    [-j <n>]         -> Render on n GPUs\n"
				   "    [-s <n>]         -> Override sample count to n\n"
				   "    [-d <w>x<h>]     -> Override image dimensions to <w>x<h>\n"
				   "    [-t <w>x<h>]     -> Override tile  dimensions to <w>x<h>\n", argv[0]);
			exit(0);
		}
		if (!strcmp(argv[i], "-j")) {
			if (next) { int n = atoi(next); opt_int("thread_override", n < 0 ? 0 : n); }
			else fprintf(stderr, "[warn] Invalid -j parameter given!\n");
		}
		if (!strcmp(argv[i], "-s")) {
			if (next) { int n = atoi(next); opt_int("samples_override", n < 1 ? 1 : n); }
			else fprintf(stderr, "[warn] Invalid -s parameter given!\n");
		}
		if (!strcmp(argv[i], "-d")) {
			int w, h;
			if (parse_dims(next, &w, &h)) { opt_set("dims_override"); opt_int("dims_width", w); opt_int("dims_height", h); }
			else fprintf(stderr, "[warn] Invalid -d parameter given!\n");
		}
		if (!strcmp(argv[i], "-t")) {
			int w, h;
			if (parse_dims(next, &w, &h)) { opt_set("tiledims_override"); opt_int("tile_width", w); opt_int("tile_height", h); }
			else fprintf(stderr, "[warn] Invalid -t parameter given!\n");
		}
		if (argv[i][0] == '-' && argv[i][1]) opt_set(argv[i] + 1);       /* args.c:207-209: any -flag is a tag */
	}
}

bool crOptionIsSet(char *key) { return key && opt_find(key) != NULL; }
char *crPathArg(void) { struct option *o = opt_find("inputFile"); return o ? o->str : NULL; }

void crDestroyOptions(void) {
	for (int i = 0; i < g_nopts; ++i) { free(g_opts[i].key); free(g_opts[i].str); }
	free(g_opts);
	g_opts = NULL; g_nopts = 0;
}

char *crGetFilePath(char *fullPath) {
	char *copy = strdup(fullPath), *out = NULL;
	if (asprintf(&out, "%s/", dirname(copy)) < 0) out = NULL;
	free(copy);
	return out;
}

/* ---- input ------------------------------------------------------------------------------------------------------- */
static char *read_stream(FILE *f, size_t *bytes) {
	size_t cap = 1 << 16, len = 0;
	char *buf = malloc(cap);
	for (;;) {
		size_t n = fread(buf + len, 1, cap - len - 1, f);
		len += n;
		if (n == 0) break;
		if (len + 1 >= cap) { cap *= 2; buf = realloc(buf, cap); }
	}
	buf[len] = '\0';
	if (bytes) *bytes = len;
	if (!len) { free(buf); return NULL; }
	return buf;
}

char *crReadFile(size_t *bytes) {
	const char *path = crPathArg();
	FILE *f = path ? fopen(path, "rb") : NULL;
	if (!f) { fprintf(stderr, "[warn] Can't access '%s'\n", path ? path : "(no input file)"); return NULL; }
	char *buf = read_stream(f, bytes);
	fclose(f);
	return buf;
}

char *crReadStdin(size_t *bytes) { return read_stream(stdin, bytes); }

/* ---- renderer ---------------------------------------------------------------------------------------------------- */
void crSetAssetPath(void) {
	free(g_asset_path);
	g_asset_path = crOptionIsSet("inputFile") ? crGetFilePath(crPathArg()) : strdup("./");
}
char *crGetAssetPath(void) { return g_asset_path; }

void crInitRenderer(void) {
	if (g_renderer) return;
	g_renderer = newRenderer();
	g_renderer->prefs.quiet = false;
	crSetAssetPath();
}

void crDestroyRenderer(void) {
	pthread_mutex_lock(&g_image_lock);
	if (g_image) { destroyTexture8(g_image); g_image = NULL; }
	pthread_mutex_unlock(&g_image_lock);
	if (g_renderer) { destroyRenderer(g_renderer); g_renderer = NULL; }
	free(g_asset_path); g_asset_path = NULL;
}

int crLoadSceneFromBuf(char *buf) {
	if (!g_renderer || !buf) return -1;
	/* the CLI overrides parsePrefs applies (sceneloader.c:425-467) */
	int W = 0, H = 0, spp = 0;
	if (crOptionIsSet("dims_override")) { W = opt_get("dims_width"); H = opt_get("dims_height"); }
	if (crOptionIsSet("samples_override")) spp = opt_get("samples_override");
	if (crOptionIsSet("tiledims_override")) {
		g_renderer->prefs.tileWidth = (unsigned)opt_get("tile_width");
		g_renderer->prefs.tileHeight = (unsigned)opt_get("tile_height");
	}
	if (loadSceneBuf(g_renderer, buf, g_asset_path ? g_asset_path : "./", &g_output, W, H, spp, 0) != 0) {
		fprintf(stderr, "[warn] Scene builder failed due to previous error.\n");
		return -1;
	}
	g_renderer->prefs.imgFilePath = g_output.file_path;
	g_renderer->prefs.imgFileName = g_output.file_name;
	g_renderer->prefs.imgCount = g_output.count;
	g_renderer->prefs.imgType = g_output.type ? png : bmp;
	int gpus = 1;                                                    /* threads = GPUs here; JSON "threads" is a CPU count */
	if (crOptionIsSet("thread_override") && opt_get("thread_override") > 0) gpus = opt_get("thread_override");
	g_renderer->prefs.threadCount = gpus;
	return 0;
}

int crLoadSceneFromFile(char *filePath) {
	/* (the reference passes the PATH to its JSON parser here, c-ray.c:117-127; the evident intent is implemented) */
	FILE *f = filePath ? fopen(filePath, "rb") : NULL;
	if (!f) return -1;
	char *buf = read_stream(f, NULL);
	fclose(f);
	if (!buf) return -1;
	if (!crOptionIsSet("inputFile")) { free(g_asset_path); g_asset_path = crGetFilePath(filePath); }
	int rc = crLoadSceneFromBuf(buf);
	free(buf);
	return rc;
}

void crStartRenderer(void) {
	if (!g_renderer) return;
	pthread_mutex_lock(&g_image_lock);
	if (g_image) { destroyTexture8(g_image); g_image = NULL; }
	pthread_mutex_unlock(&g_image_lock);
	struct texture8 *img = renderFrame(g_renderer);                  /* c-ray.c:257 */
	if (!img) fprintf(stderr, "[ERR ] render failed: %s\n", crgpu_last_error());
	pthread_mutex_lock(&g_image_lock);
	if (g_image) destroyTexture8(g_image);                           /* taken by crGetCurrentImage during the frame */
	g_image = img;
	pthread_mutex_unlock(&g_image_lock);
}

static void write_image_locked(void);
void crWriteImage(void) {
	pthread_mutex_lock(&g_image_lock);
	write_image_locked();
	pthread_mutex_unlock(&g_image_lock);
}
static void write_image_locked(void) {                               /* c-ray.c:77-98, encoder.c:22-39 */
	if (!g_image || !g_renderer) return;
	char *path = NULL;
	if (asprintf(&path, "%s%s_%04d.%s", g_renderer->prefs.imgFilePath, g_renderer->prefs.imgFileName, g_renderer->prefs.imgCount,
				 g_renderer->prefs.imgType == png ? "png" : "bmp") < 0) return;
	struct renderInfo info;
	rendererInfo(g_renderer, &info);
	if (writeImageInfo(g_image, path, g_renderer->prefs.imgType, &info) != 0) {
		/* fileio.c:93-109: fall back to the working directory when the output directory is not writable */
		char *fallback = NULL;
		if (asprintf(&fallback, "./%s_%04d.%s", g_renderer->prefs.imgFileName, g_renderer->prefs.imgCount,
					 g_renderer->prefs.imgType == png ? "png" : "bmp") >= 0 && writeImageInfo(g_image, fallback, g_renderer->prefs.imgType, &info) == 0)
			printf("[info] Saving result in \"%s\"\n", fallback);
		else fprintf(stderr, "[warn] Image can't be saved to \"%s\"\n", path);
		free(fallback);
	} else printf("[info] Saving result in \"%s\"\n", path);
	free(path);
}

/* ---- prefs ------------------------------------------------------------------------------------------------------- */
static void reconfigure(int w, int h, int spp, int bounces) {
	if (g_renderer && g_renderer->scene.prefs.image_width) applySceneConfig(g_renderer, w, h, spp, bounces);
}
void crSetThreadCount(int threadCount, bool fromSystem) { (void)fromSystem; if (g_renderer && threadCount > 0) g_renderer->prefs.threadCount = threadCount; }
int crGetThreadCount(void) { return g_renderer ? g_renderer->prefs.threadCount : 0; }
void crSetSampleCount(int sampleCount) { if (sampleCount > 0) reconfigure(0, 0, sampleCount, 0); }
int crGetSampleCount(void) { return g_renderer ? g_renderer->prefs.sampleCount : 0; }
void crSetBounces(int bounces) { if (bounces > 0) reconfigure(0, 0, 0, bounces); }
int crGetBounces(void) { return g_renderer ? g_renderer->prefs.bounces : 0; }
void crSetTileWidth(unsigned width) { if (g_renderer && width > 0) { g_renderer->prefs.tileWidth = width; reconfigure(0, 0, 0, 0); } }
unsigned crGetTileWidth(void) { return g_renderer ? g_renderer->prefs.tileWidth : 0; }
void crSetTileHeight(unsigned height) { if (g_renderer && height > 0) { g_renderer->prefs.tileHeight = height; reconfigure(0, 0, 0, 0); } }
unsigned crGetTileHeight(void) { return g_renderer ? g_renderer->prefs.tileHeight : 0; }
void crSetImageWidth(unsigned width) { if (g_renderer && width > 0) reconfigure((int)width, (int)g_renderer->prefs.imageHeight, 0, 0); }
unsigned crGetImageWidth(void) { return g_renderer ? g_renderer->prefs.imageWidth : 0; }
void crSetImageHeight(unsigned height) { if (g_renderer && height > 0) reconfigure((int)g_renderer->prefs.imageWidth, (int)height, 0, 0); }
unsigned crGetImageHeight(void) { return g_renderer ? g_renderer->prefs.imageHeight : 0; }
void crSetOutputPath(char *filePath) { if (g_renderer && filePath) { snprintf(g_output.file_path, sizeof(g_output.file_path), "%s", filePath); g_renderer->prefs.imgFilePath = g_output.file_path; } }
char *crGetOutputPath(void) { return g_renderer ? (char *)g_renderer->prefs.imgFilePath : NULL; }
void crSetFileName(char *fileName) { if (g_renderer && fileName) { snprintf(g_output.file_name, sizeof(g_output.file_name), "%s", fileName); g_renderer->prefs.imgFileName = g_output.file_name; } }
char *crGetFileName(void) { return g_renderer ? (char *)g_renderer->prefs.imgFileName : NULL; }
void crSetAntialiasing(bool on) { g_antialiasing = on; }               /* stored only: the reference's renderThread never reads it either */
bool crGetAntialiasing(void) { return g_antialiasing; }

/* ---- not implemented by the reference either ------------------------------------------------------------------------ */
static void not_available(const char *what) { fprintf(stderr, "[warn] %s is not available on the GPU path\n", what); }
void crLoadMeshFromFile(char *filePath) { (void)filePath; not_available("crLoadMeshFromFile"); }
void crLoadMeshFromBuf(char *buf) { (void)buf; not_available("crLoadMeshFromBuf"); }
void crSetRenderOrder(void) { not_available("crSetRenderOrder"); }
void crGetRenderOrder(void) { not_available("crGetRenderOrder"); }
void crStartRenderWorker(void) { not_available("the network render worker (src/utils/protocol/worker.c)"); }
void crStartInteractive(void) { not_available("crStartInteractive"); }
void crPauseInteractive(void) { not_available("crPauseInteractive"); }
/* "Just get the current buffer" (src/c-ray.h:97): the current image becomes the frame as it stands (crhostCurrentImage), from any
 * thread, so that crWriteImage writes what a frame in flight shows at this moment */
void crGetCurrentImage(void) {
	if (!g_renderer || !g_renderer->prefs.imageWidth) return;
	const unsigned W = g_renderer->prefs.imageWidth, H = g_renderer->prefs.imageHeight;
	pthread_mutex_lock(&g_image_lock);
	if (g_image && (g_image->width != W || g_image->height != H)) { destroyTexture8(g_image); g_image = NULL; }
	if (!g_image) {
		g_image = calloc(1, sizeof *g_image);
		if (g_image) { g_image->width = W; g_image->height = H; g_image->data = malloc((size_t)W * H * 3); }
		if (g_image && !g_image->data) { free(g_image); g_image = NULL; }
	}
	if (g_image) crhostCurrentImage(g_renderer, g_image->data);
	pthread_mutex_unlock(&g_image_lock);
}
void crRestartInteractive(void) { }

/* ---- additions ----------------------------------------------------------------------------------------------------- */
const float *crGetRenderBuffer(unsigned *width, unsigned *height) {
	if (!g_renderer || !g_image) return NULL;
	if (width) *width = g_renderer->prefs.imageWidth;
	if (height) *height = g_renderer->prefs.imageHeight;
	return g_renderer->state.renderBuffer;
}
double crGetRenderSeconds(void) { return g_renderer ? g_renderer->state.renderSeconds : 0.0; }
unsigned long long crGetRayCount(void) { return g_renderer ? (unsigned long long)g_renderer->state.totalRays : 0ull; }
