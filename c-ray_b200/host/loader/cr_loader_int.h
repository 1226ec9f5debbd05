/*
 * cr_loader_int.h — internal structures shared by the pieces of the scene loader (c-ray_b200/host/loader/).
 *
 * The loader is the host-side "next row" after the hot path (SURVEY.md §8 f2): it turns a c-ray JSON scene + its
 * OBJ/MTL/PNG/HDR assets into the flat `struct crs_scene` of include/crscene.h, so that `cray_b200 scene.json`
 * works without the reference.  Target behaviour = what the reference's own loader produces for the same files
 * (src/utils/loaders/sceneloader.c, formats/wavefront/, textureloader.c, src/accelerators/bvh.c), checked array by
 * array against `oracle/_ref/cray_ref_strict export` in tests/test_loader.py.
 */
#pragma once
#include <stdint.h>
#include <stddef.h>
#include "../../../include/crscene.h"
#include "cr_math.h"
#include "cr_image.h"

enum crl_bsdf_type { CRL_EMISSION = 0, CRL_LAMBERTIAN, CRL_GLASS, CRL_PLASTIC, CRL_METAL };   /* material.h:52-60 */

struct crl_color { float r, g, b, a; };

struct crl_material {             /* the fields of reference struct material the loader touches (material.h:62-83) */
	char *name;
	struct crl_color diffuse, specular, emission;
	int illum;
	float IOR, roughness;
	enum crl_bsdf_type type;
	int texture, specular_map;    /* loader texture handles, -1 = none */
	int bsdf;                     /* loader node handle, -1 = none */
};

struct crl_mesh {
	struct crs_poly *polys;       /* indices already global (wavefront.c:119-125) */
	int poly_count;
	struct crl_material *materials;
	int material_count;
	int texcoord_count;           /* vt lines of THIS file (mesh->textureCoordCount) */
	float ray_offset;
	struct crs_bvh_node *bvh_nodes;
	int32_t *bvh_prims;
	uint32_t bvh_node_count;
};

struct crl_sphere {
	float radius, ray_offset;
	struct crl_material material;
};

struct crl_instance {
	struct xform composite;
	int is_mesh;
	int object;
};

struct crl_node {                 /* one hash-consed node; inputs are loader node handles */
	int kind;
	int in[3];
	float f[8];
	int tex;
	uint32_t options;
};

struct crl_ctx {
	char *asset_path;             /* directory of the JSON file + "/" (c-ray.c:255) */
	char err[512];

	/* global vertex buffers (vertexbuffer.c:14-21) */
	float *vertices, *normals, *texcoords;
	int vertex_count, normal_count, texcoord_count;

	struct cr_image *textures;    /* every successful loadTexture() call, in call order */
	int texture_count;
	/* texture files are decoded on background threads while parsing and BVH construction go on (a 2048x2048 PNG inflates
	 * for ~0.1 s on one core); a decode that fails after its header looked fine makes the whole load restart synchronously,
	 * because a missing texture changes the node graph (image.c:51: NULL texture -> no image node) */
	struct crl_tex_job **tex_jobs;
	int async_textures, async_failed;

	struct crl_node *nodes;       /* creation order */
	int node_count, node_cap;

	struct crl_mesh *meshes;      int mesh_count;
	struct crl_sphere *spheres;   int sphere_count;
	struct crl_instance *instances; int instance_count, instance_cap;
	int background;
};

/* cr_wavefront.c */
int crl_load_obj(struct crl_ctx *c, const char *path, struct crl_mesh *out);      /* 0 ok, 1 = "no mesh" (skip), <0 error */
int crl_load_texture(struct crl_ctx *c, const char *path);                        /* handle or -1 */
void crl_textures_join(struct crl_ctx *c);                                        /* waits for background decodes; sets c->async_failed */

/* cr_bvh_build.c */
typedef void (*crl_bbox_fn)(void *user, unsigned i, bbox3 *bbox, vec3 *center);
int crl_build_bvh(void *user, crl_bbox_fn fn, unsigned count,
                  struct crs_bvh_node **nodes, uint32_t *node_count, int32_t **prims);

/* cr_sceneload.c: the message of crloader_last_error() */
void crl_set_error(const char *fmt, ...) __attribute__((format(printf, 1, 2)));

/* cr_threads.c */
int crl_thread_count(void);
void crl_parallel_for(int n, void (*fn)(void *arg, int index), void *arg);

/* cr_nodes.c */
int crl_const_color(struct crl_ctx *c, struct crl_color col);
int crl_image(struct crl_ctx *c, int tex, uint32_t options);                      /* -1 when tex < 0 (image.c:51) */
int crl_checker(struct crl_ctx *c, int A, int B, int scale);
int crl_gradient(struct crl_ctx *c, struct crl_color down, struct crl_color up);
int crl_blackbody(struct crl_ctx *c, int temperature);
int crl_const_value(struct crl_ctx *c, float v);
int crl_grayscale(struct crl_ctx *c, int color);
int crl_alpha(struct crl_ctx *c, int color);
int crl_diffuse(struct crl_ctx *c, int color);
int crl_metal(struct crl_ctx *c, int color, int roughness);
int crl_glass(struct crl_ctx *c, int color, int roughness, int ior);
int crl_plastic(struct crl_ctx *c, int color);
int crl_mix(struct crl_ctx *c, int A, int B, int factor);
int crl_add(struct crl_ctx *c, int A, int B);
int crl_transparent(struct crl_ctx *c, int color);
int crl_emissive(struct crl_ctx *c, int color, int strength);
int crl_background(struct crl_ctx *c, int color, int strength, int offset);
int crl_warning_bsdf(struct crl_ctx *c);
void crl_assign_bsdf(struct crl_ctx *c, struct crl_material *m);

extern const struct crl_color crl_black, crl_white, crl_gray;
