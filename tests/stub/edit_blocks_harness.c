/* tests/stub/edit_blocks_harness.c — the device blocks of the resident-scene edits against the CUDA stub (tests/stub/cudart_stub.c),
 * linked with -fsanitize=address.  Usage: edit_blocks_harness A.crscene SHADE.crscene B1.crscene B2.crscene
 *
 * Two scenes g and h are created from A and take the same edits, each one that needs no kernel result: set_camera, set_views (grow,
 * shrink, grow again), set_render (with a resize and without), set_shading (SHADE: A's material count), set_instance_list with no
 * instances, and add_objects of B1 and then B2.  h takes each edit once.  g takes it with cudaMalloc failing from its k-th call on,
 * for k = 1, 2, ... until the call succeeds: every failed call must return CRGPU_ERR_NOMEM and leave g's observable state as it was,
 * and the call that succeeds must leave g in h's state.  The per-device cache is trimmed after every call, so that a block the scene
 * still uses is back in malloc's hands, where ASan reports the next read of it.  Prints one "op <name> allocs <k>" line per edit,
 * then "live <n>": the device allocations left after both scenes are destroyed and the cache trimmed. */
#include "crgpu.h"
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <stdint.h>

long stub_live_allocs(void);
void stub_fail_malloc_from(long k);

static struct crs_scene A, SHADE, B1, B2;
static struct crs_camera cams[4];

static void die(const char *what, int rc) {
	printf("FAIL %s rc=%d (%s)\n", what, rc, crgpu_last_error());
	exit(1);
}

/* FNV-1a over everything an edit may change that the API shows: shading, view count, image size and every view's pixels */
static uint64_t fnv(uint64_t h, const void *p, size_t n) {
	const unsigned char *b = p;
	for (size_t i = 0; i < n; ++i) h = (h ^ b[i]) * 1099511628211ull;
	return h;
}
static uint64_t state(crgpu_scene *g) {
	uint64_t h = 1469598103934665603ull;
	uint32_t n = 0, bg = 0, views = 0;
	int x = 0, dev = 0, w = 0, ht = 0, rc;
	if ((rc = crgpu_scene_shading(g, NULL, NULL, 0, &n, &bg, &x))) die("shading", rc);
	uint32_t *k = calloc(2 * (size_t)n + 1, 4);
	if ((rc = crgpu_scene_shading(g, k, k + n, n, NULL, NULL, NULL))) die("shading", rc);
	h = fnv(h, &n, 4); h = fnv(h, &bg, 4); h = fnv(h, &x, 4); h = fnv(h, k, 8 * (size_t)n);
	free(k);
	if ((rc = crgpu_scene_view_count(g, &views))) die("view_count", rc);
	if ((rc = crgpu_scene_info(g, &dev, &w, &ht))) die("info", rc);
	h = fnv(h, &views, 4); h = fnv(h, &w, 4); h = fnv(h, &ht, 4);
	float *px = malloc((size_t)w * ht * 3 * sizeof(float));
	uint8_t *rgb8 = malloc((size_t)w * ht * 3);
	for (uint32_t v = 0; v < views; ++v) {
		if ((rc = crgpu_view_read(g, v, px))) die("view_read", rc);
		h = fnv(h, px, (size_t)w * ht * 3 * sizeof(float));
	}
	/* the sRGB8 staging at the current size (its bytes are no kernel's: not hashed) */
	if ((rc = crgpu_framebuffer_to_srgb8(g, rgb8)) || (rc = crgpu_view_to_srgb8(g, views - 1u, rgb8))) die("to_srgb8", rc);
	free(px);
	free(rgb8);
	crgpu_device_trim(0);
	return h;
}

/* view 0's pixels: the only ones a test without kernels can give values */
static void paint(crgpu_scene *g) {
	int dev = 0, w = 0, h = 0, rc;
	crgpu_scene_info(g, &dev, &w, &h);
	float *px = malloc((size_t)w * h * 3 * sizeof(float));
	for (size_t i = 0; i < (size_t)w * h * 3; ++i) px[i] = (float)i * 0.25f;
	if ((rc = crgpu_framebuffer_write(g, px, 0, 0, 0, 0))) die("framebuffer_write", rc);
	free(px);
	crgpu_device_trim(0);
}

static const char *const OPS[] = { "set_camera", "set_views_3", "set_views_2", "set_views_4", "set_render_resize", "set_render",
                                   "set_shading", "set_instance_list_empty", "add_objects_sphere", "add_objects_empty_mesh" };
enum { NOPS = sizeof OPS / sizeof OPS[0] };

static int run(int op, crgpu_scene *g) {
	switch (op) {
	case 0: return crgpu_scene_set_camera(g, &cams[1]);
	case 1: return crgpu_scene_set_views(g, cams, 3);
	case 2: return crgpu_scene_set_views(g, cams, 2);
	case 3: return crgpu_scene_set_views(g, cams, 4);
	case 4: {
		struct crs_camera c[4];
		memcpy(c, cams, sizeof c);
		for (int i = 0; i < 4; ++i) { c[i].width = 24; c[i].height = 10; }
		return crgpu_scene_set_render(g, 24, 10, 2, 3, c, 4);
	}
	case 5: return crgpu_scene_set_render(g, 24, 10, 3, 1, NULL, 4);
	case 6: return crgpu_scene_set_shading(g, &SHADE);
	case 7: return crgpu_scene_set_instance_list(g, NULL, 0);
	case 8: return crgpu_scene_add_objects(g, &B1);
	default: return crgpu_scene_add_objects(g, &B2);
	}
}

int main(int argc, char **argv) {
	if (argc < 5) return 2;
	if (crscene_load(&A, argv[1]) || crscene_load(&SHADE, argv[2]) || crscene_load(&B1, argv[3]) || crscene_load(&B2, argv[4])) return 1;
	crscene_set_config(&A, 16, 8, 1, 2);
	for (int i = 0; i < 4; ++i) { cams[i] = A.camera; cams[i].focal_distance += (float)i; }
	crgpu_scene *g = NULL, *h = NULL;
	int rc;
	if ((rc = crgpu_scene_create(&A, 0, &g)) || (rc = crgpu_scene_create(&A, 0, &h))) die("create", rc);
	paint(g);
	paint(h);
	for (int op = 0; op < NOPS; ++op) {
		if ((rc = run(op, h))) die(OPS[op], rc);
		crgpu_device_trim(0);
		if (op == 4) paint(h);
		const uint64_t want = state(h), before = state(g);
		long k = 1;
		for (;; ++k) {
			stub_fail_malloc_from(k);
			rc = run(op, g);
			stub_fail_malloc_from(-1);
			crgpu_device_trim(0);
			if (rc == CRGPU_OK) break;
			if (rc != CRGPU_ERR_NOMEM) { printf("FAIL %s allocation %ld: rc=%d (%s)\n", OPS[op], k, rc, crgpu_last_error()); return 1; }
			if (state(g) != before) { printf("FAIL %s allocation %ld: the failed call changed the scene\n", OPS[op], k); return 1; }
			if (k > 64) { printf("FAIL %s: no success after %ld allocations\n", OPS[op], k); return 1; }
		}
		if (op == 4) paint(g);
		if (state(g) != want) { printf("FAIL %s: the scene differs from the one the call made unfailed\n", OPS[op]); return 1; }
		printf("op %s allocs %ld\n", OPS[op], k - 1);
	}
	crgpu_scene_destroy(g);
	crgpu_scene_destroy(h);
	crgpu_device_trim(0);
	printf("live %ld\n", stub_live_allocs());
	crscene_free(&A);
	crscene_free(&SHADE);
	crscene_free(&B1);
	crscene_free(&B2);
	return 0;
}
