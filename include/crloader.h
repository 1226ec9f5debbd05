/*
 * crloader.h — the scene loader's C ABI (c-ray_b200/libcrloader.so, sources in c-ray_b200/host/loader/).
 *
 * Builds the flat scene of crscene.h straight from a c-ray JSON scene file and the OBJ/MTL/PNG/HDR assets it names:
 * the job of the reference's loadScene (reference src/datatypes/scene.c:121-212 -> parseJSON,
 * src/utils/loaders/sceneloader.c:1153-1203) including both BVH levels (src/accelerators/bvh.c:245-315).
 * Pure host C (zlib + libm), no CUDA: the result is handed to crgpu_scene_create (crgpu.h) or crscene_save.
 *
 * Asset paths resolve like the reference's: meshes and the HDR environment relative to the JSON file
 * (sceneloader.c:698,905), textures named inside node graphs relative to the working directory (:783,:826).
 */
#pragma once
#include "crscene.h"

#ifdef __cplusplus
extern "C" {
#endif

/* 0 on success, negative on error (message in crloader_last_error()).  Release with crscene_free (or free(out->owner)).
 * CLI-style overrides (-d WxH, -s N) are applied afterwards with crscene_set_config, which is arithmetically the
 * same as the reference applying them before newCamera (sceneloader.c:425-467, camera.c:22-42). */
int crloader_load_json(struct crs_scene *out, const char *json_path);

/* Where and how the reference would save the frame: "renderer".outputFilePath / outputFileName / count / fileType
 * (sceneloader.c:341-424); the file is <file_path><file_name>_<count %04d>.<png|bmp> (src/utils/encoders/encoder.c:24). */
struct crloader_output {
	char file_path[512];
	char file_name[256];
	int  count;
	int  type;                 /* 0 = bmp, 1 = png (enum fileType) */
};

/* Same, from JSON text already in memory (crLoadSceneFromBuf, reference src/c-ray.c:139-141); `asset_path` is the
 * directory prefix (with trailing '/') mesh and HDR names are appended to, NULL = "./"; `output` may be NULL. */
int crloader_load_json_buf(struct crs_scene *out, const char *json_text, const char *asset_path, struct crloader_output *output);
const char *crloader_last_error(void);

/* The BVH builder on its own (reference src/accelerators/bvh.c:245-296 buildBvhGeneric): n primitives given by their boxes
 * (n x 6 floats: min.xyz, max.xyz) and centers (n x 3); nodes_out has room for 2n-1 nodes, prims_out for n indices.
 * Host counterpart of crgpu_bvh_build (crgpu.h, SURVEY 8 f1), same outputs bit for bit.  0 on success.
 * A tree can need more than 2n-1 nodes: 17 or more primitives that no split separates (centres at one point, or a node whose extent
 * overflows to inf) take the median fallback, which sends all of them left, so each such node gets an empty right leaf (count 0,
 * the empty box) and a left child with the same primitives, down to depth 64.  Then nothing is written to nodes_out or prims_out,
 * *node_count_out is set to the number of nodes the tree needs and -2 is returned.  crloader_load_json* store such trees whole. */
int crloader_build_bvh(const float *bboxes, const float *centers, uint32_t n,
                       struct crs_bvh_node *nodes_out, uint32_t *node_count_out, int32_t *prims_out);

/* Route the BVH builds of crloader_load_json* through another builder with crloader_build_bvh's signature (e.g. a wrapper of
 * crgpu_bvh_build) for inputs of at least `min_prims` primitives; NULL restores the host builder.  A builder that returns
 * non-zero falls back to the host builder for that BVH.  Process-wide; set it before loading. */
typedef int (*crloader_bvh_builder)(const float *bboxes, const float *centers, uint32_t n,
                                    struct crs_bvh_node *nodes_out, uint32_t *node_count_out, int32_t *prims_out);
void crloader_set_bvh_builder(crloader_bvh_builder fn, uint32_t min_prims);

#ifdef __cplusplus
}
#endif
