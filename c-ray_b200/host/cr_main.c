/*
 * cr_main.c — command-line driver of the host mirror: cray_b200 <scene.json | scene.crscene> [options]
 *
 * The counterpart of reference src/main.c:14-42 for this path: load → renderFrame → writeImage.  The scene
 * is either a c-ray JSON scene (parsed and BVH-built by the host loader, c-ray_b200/host/loader/) or a
 * flattened .crscene (include/crscene.h); the CLI
 * overrides mirror the reference's (-d WxH, -s N, -t WxH, -j N: src/utils/args.c:95-142), with -j counting
 * GPUs instead of CPU threads and -b for the bounce limit the reference only takes from the JSON.
 */
#include "cr_host.h"
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <math.h>

static int parse_dims(const char *s, int *w, int *h) { return s && sscanf(s, "%dx%d", w, h) == 2 && *w > 0 && *h > 0; }

int main(int argc, char **argv) {
	if (argc < 2) {
		fprintf(stderr, "usage: %s scene.json|scene.crscene [-d WxH] [-s samples] [-b bounces] [-t tileWxtileH] [-j gpus] [-o out.png|out.bmp] [--dump-f32 file] [--adaptive threshold] [--dump-passes file] [--gpu-bvh] [-q]\n", argv[0]);
		return 1;
	}
	int W = 0, H = 0, spp = 0, bounces = 0, tw = 0, th = 0, gpus = 1, quiet = 0;
	const char *out = NULL, *dump = NULL, *dump_passes = NULL;
	float threshold = 0.f;
	int adaptive = 0;
	for (int i = 2; i < argc; ++i) {
		if (!strcmp(argv[i], "-d") && i + 1 < argc) { if (!parse_dims(argv[++i], &W, &H)) { fprintf(stderr, "Invalid -d parameter given!\n"); return 1; } }
		else if (!strcmp(argv[i], "-s") && i + 1 < argc) spp = atoi(argv[++i]);
		else if (!strcmp(argv[i], "-b") && i + 1 < argc) bounces = atoi(argv[++i]);
		else if (!strcmp(argv[i], "-t") && i + 1 < argc) { if (!parse_dims(argv[++i], &tw, &th)) { fprintf(stderr, "Invalid -t parameter given!\n"); return 1; } }
		else if (!strcmp(argv[i], "-j") && i + 1 < argc) gpus = atoi(argv[++i]);
		else if (!strcmp(argv[i], "-o") && i + 1 < argc) out = argv[++i];
		else if (!strcmp(argv[i], "--dump-f32") && i + 1 < argc) dump = argv[++i];
		else if (!strcmp(argv[i], "--adaptive") && i + 1 < argc) {
			/* stop sampling a pixel once its error estimate is below the threshold (crhostSetAdaptive) */
			char *end = NULL;
			const char *v = argv[++i];
			threshold = strtof(v, &end);
			if (end == v || *end || !isfinite(threshold) || threshold < 0.f) { fprintf(stderr, "Invalid --adaptive parameter given: %s\n", v); return 1; }
			adaptive = 1;
		}
		else if (!strcmp(argv[i], "--dump-passes") && i + 1 < argc) dump_passes = argv[++i];
		else if (!strcmp(argv[i], "-q")) quiet = 1;
		else if (!strcmp(argv[i], "--gpu-bvh")) crhostUseGpuBvh(1, 0, 1024);      /* SURVEY 8(f1): BVHs of >= 1024 primitives built on device 0 */
		else { fprintf(stderr, "unknown option %s\n", argv[i]); return 1; }
	}
	struct renderer *r = newRenderer();
	r->prefs.threadCount = gpus < 1 ? 1 : gpus;
	r->prefs.tileWidth = (unsigned)tw; r->prefs.tileHeight = (unsigned)th;
	r->prefs.quiet = quiet != 0;
	if (adaptive) crhostSetAdaptive(r, 1, threshold);
	if (loadSceneFile(r, argv[1], W, H, spp, bounces) != 0) { fprintf(stderr, "cannot load %s\n", argv[1]); destroyRenderer(r); return 2; }
	struct texture8 *img = renderFrame(r);
	if (!img) { destroyRenderer(r); return 3; }
	int rc = 0;
	if (out) {
		const size_t n = strlen(out);
		const enum fileType ft = (n > 4 && !strcmp(out + n - 4, ".bmp")) ? bmp : png;
		struct renderInfo info;
		rendererInfo(r, &info);
		if (writeImageInfo(img, out, ft, &info) != 0) { fprintf(stderr, "cannot write %s\n", out); rc = 4; }
		else if (!quiet) printf("Saved result to %s\n", out);
	}
	if (dump) {
		FILE *f = fopen(dump, "wb");
		if (f) { fwrite(r->state.renderBuffer, sizeof(float), (size_t)r->prefs.imageWidth * r->prefs.imageHeight * 3, f); fclose(f); } else rc = 4;
	}
	if (dump_passes) {           /* raw u32 pass counts, W*H, rows top to bottom as in the framebuffer (an adaptive frame only) */
		const uint32_t *p = crhostAdaptivePasses(r);
		FILE *f = p ? fopen(dump_passes, "wb") : NULL;
		if (f) { fwrite(p, sizeof(uint32_t), (size_t)r->prefs.imageWidth * r->prefs.imageHeight, f); fclose(f); }
		else { fprintf(stderr, "cannot write %s%s\n", dump_passes, p ? "" : ": --dump-passes needs --adaptive"); rc = 4; }
	}
	destroyTexture8(img);
	destroyRenderer(r);
	return rc;
}
