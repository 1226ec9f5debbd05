/* tests/stub/shading_harness.c — crgpu_scene_set_shading against the CUDA stub: scene A.crscene takes the shading of B.crscene.
 * Prints crgpu_prepare's code for B, set_shading's code, and crgpu_scene_shading of A before and after the edit, of a scene created
 * fresh from B's prepare, and B's prepared queries (kinds, flags, background kind; "x" = complete interpreter). */
#include "crgpu.h"
#include <stdio.h>
#include <stdlib.h>
#include <stdint.h>

static void show(const char *what, crgpu_scene *g) {
	uint32_t n = 0, bg = 0; int x = 0;
	crgpu_scene_shading(g, NULL, NULL, 0, &n, &bg, &x);
	uint32_t *k = calloc(n + 1, 4), *f = calloc(n + 1, 4);
	crgpu_scene_shading(g, k, f, n, NULL, NULL, NULL);
	printf("%s n=%u bg=%u x=%d", what, n, bg, x);
	for (uint32_t i = 0; i < n; ++i) printf(" %u/%u", k[i], f[i]);
	printf("\n");
	free(k); free(f);
}

int main(int argc, char **argv) {
	if (argc < 3) return 2;
	struct crs_scene a, b;
	if (crscene_load(&a, argv[1]) || crscene_load(&b, argv[2])) return 1;
	crscene_set_config(&a, 32, 32, 1, 4);
	crscene_set_config(&b, 32, 32, 1, 4);
	crgpu_scene *g = NULL, *fresh = NULL;
	if (crgpu_scene_create(&a, 0, &g)) { printf("create A failed: %s\n", crgpu_last_error()); return 1; }
	crgpu_prepared *p = NULL;
	int prc = crgpu_prepare(&b, &p);
	printf("prepare rc=%d\n", prc);
	show("before", g);
	int src = crgpu_scene_set_shading(g, &b);
	printf("set rc=%d (%s)\n", src, src ? crgpu_last_error() : "ok");
	show("edited", g);
	if (!prc) {
		uint32_t n = 0, bg = 0;
		crgpu_prepared_materials(p, NULL, NULL, 0, &n);
		uint32_t *k = calloc(n + 1, 4), *f = calloc(n + 1, 4);
		crgpu_prepared_materials(p, k, f, n, NULL);
		crgpu_prepared_background(p, &bg);
		printf("prepared n=%u bg=%u", n, bg);
		for (uint32_t i = 0; i < n; ++i) printf(" %u/%u", k[i], f[i]);
		printf("\n");
		free(k); free(f);
		if (!crgpu_scene_create_prepared(p, 0, &fresh)) show("fresh", fresh);
		crgpu_scene_destroy(fresh);
		crgpu_prepared_free(p);
	}
	crgpu_scene_destroy(g);
	crscene_free(&a);
	crscene_free(&b);
	return 0;
}
