/*
 * cr_sceneload.c — c-ray JSON scene -> flat `struct crs_scene` (crloader_load_json, include/crloader.h).
 *
 * Follows the reference loader statement by statement where the result depends on it
 * (reference src/utils/loaders/sceneloader.c): prefs with their defaults and clamps (:190-424), camera (:547-626 +
 * src/datatypes/camera.c:22-42), colours (:628-678), ambient colour / HDR environment (:681-713), transform lists
 * folded as translates, then rotates, then scales (:716-755), node graphs (:765-875), meshes with their instances
 * and legacy or graph materials (:878-990), spheres (:1008-1100).  After parsing, the two-level BVH is built
 * (src/datatypes/scene.c:184-185; ray offsets are a side effect of the top-level build, instance.c:94-110,:221-230)
 * and everything is flattened in the order of oracle/ref_harness.c's flatten(), so the two can be compared
 * array by array (tests/test_loader.py).
 * Volumes ("density") are not created by the reference's JSON loader either.
 */
#include "cr_loader_int.h"
#include "cr_json.h"
#include "../../../include/crloader.h"
#include <stdarg.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <libgen.h>
#include <unistd.h>

static _Thread_local char g_err[512];
const char *crloader_last_error(void) { return g_err; }
void crl_set_error(const char *fmt, ...) {
	va_list ap;
	va_start(ap, fmt);
	vsnprintf(g_err, sizeof(g_err), fmt, ap);
	va_end(ap);
}

/* ---- small helpers ------------------------------------------------------------------------------------- */
static char *slurp(const char *path) {
	FILE *f = fopen(path, "rb");
	if (!f) return NULL;
	fseek(f, 0, SEEK_END);
	long n = ftell(f);
	fseek(f, 0, SEEK_SET);
	char *buf = n > 0 ? malloc((size_t)n + 1) : NULL;
	if (buf && fread(buf, 1, (size_t)n, f) == (size_t)n) buf[n] = '\0'; else { free(buf); buf = NULL; }
	fclose(f);
	return buf;
}

static int file_exists(const char *p) { FILE *f = fopen(p, "r"); if (f) fclose(f); return f != NULL; }

static char *join(const char *a, const char *b) {
	char *s = malloc(strlen(a) + strlen(b) + 1);
	strcpy(s, a); strcat(s, b);
	return s;
}

static int str_eq(const struct crj *j, const char *s) { return crj_is_string(j) && !strcmp(j->str, s); }

/* ---- colours ------------------------------------------------------------------------------------------- */
static struct crl_color kelvin_color(float kelvin) {                       /* src/datatypes/color.c:28-70 */
	float red, green, blue;
	float temp = kelvin >= 40000.0f ? 40000.0f : kelvin;
	temp = temp / 100.0f;
	if (temp <= 66.0f) red = 255.0f;
	else {
		red = temp - 60.0f;
		red = 329.698727446f * powf(red, -0.1332047592f);
		red = red < 0.0f ? 0.0f : red;
		red = red > 255.0f ? 255.0f : red;
	}
	if (temp <= 66.0f) {
		green = temp;
		green = 99.4708025861f * logf(green) - 161.1195681661f;
	} else {
		green = temp - 60.0f;
		green = 288.1221695283f * powf(green, -0.0755148492f);
	}
	green = green < 0.0f ? 0.0f : green;
	green = green > 255.0f ? 255.0f : green;
	if (temp >= 66.0f) blue = 255.0f;
	else if (temp <= 19.0f) blue = 0.0f;
	else {
		blue = temp - 10.0f;
		blue = 138.5177312231f * logf(blue) - 305.0447927307f;
		blue = blue < 0.0f ? 0.0f : blue;
		blue = blue > 255.0f ? 255.0f : blue;
	}
	return (struct crl_color){ red / 255.0f, green / 255.0f, blue / 255.0f, 0 };
}

static float num_or(const struct crj *j, float def) { return crj_is_number(j) ? (float)j->num : def; }

static struct crl_color parse_color(const struct crj *d) {
	if (crj_is_array(d))
		return (struct crl_color){ num_or(crj_at(d, 0), 0.0f), num_or(crj_at(d, 1), 0.0f), num_or(crj_at(d, 2), 0.0f), num_or(crj_at(d, 3), 1.0f) };
	const struct crj *k = crj_get(d, "blackbody");
	if (crj_is_number(k)) return kelvin_color((float)k->num);
	return (struct crl_color){ num_or(crj_get(d, "r"), 0.0f), num_or(crj_get(d, "g"), 0.0f), num_or(crj_get(d, "b"), 0.0f), num_or(crj_get(d, "a"), 1.0f) };
}

static struct crl_color color_coef(float k, struct crl_color c) { return (struct crl_color){ c.r * k, c.g * k, c.b * k, c.a * k }; }

/* ---- transforms ---------------------------------------------------------------------------------------- */
static struct xform parse_transform(const struct crj *d) {
	const struct crj *type = crj_get(d, "type");
	const char *t = crj_is_string(type) ? type->str : "";
	const struct crj *degrees = crj_get(d, "degrees"), *radians = crj_get(d, "radians"), *scale = crj_get(d, "scale");
	const struct crj *X = crj_get(d, "X"), *Y = crj_get(d, "Y"), *Z = crj_get(d, "Z");
	float def = !strcmp(t, "scale") ? 1.0f : 0.0f;
	int valid = 0;
	float x = def, y = def, z = def;
	if (crj_is_number(X)) { x = (float)X->num; valid++; }
	if (crj_is_number(Y)) { y = (float)Y->num; valid++; }
	if (crj_is_number(Z)) { z = (float)Z->num; valid++; }
	const int rot = !strcmp(t, "rotateX") ? 0 : !strcmp(t, "rotateY") ? 1 : !strcmp(t, "rotateZ") ? 2 : -1;
	if (rot >= 0) {
		float rads = 0.0f;
		int ok = 1;
		if (crj_is_number(degrees)) rads = crl_to_radians((float)degrees->num);
		else if (crj_is_number(radians)) rads = (float)radians->num;
		else ok = 0;
		if (ok) return rot == 0 ? crl_xf_rotate_x(rads) : rot == 1 ? crl_xf_rotate_y(rads) : crl_xf_rotate_z(rads);
	} else if (!strcmp(t, "translate")) {
		if (valid > 0) return crl_xf_translate(x, y, z);
	} else if (!strcmp(t, "scale")) {
		if (valid > 0) return crl_xf_scale(x, y, z);
	} else if (!strcmp(t, "scaleUniform")) {
		if (crj_is_number(scale)) { float s = (float)scale->num; return crl_xf_scale(s, s, s); }
	}
	fprintf(stderr, "cr_loader: ignoring invalid transform \"%s\"\n", t);
	return crl_xf_translate(0.0f, 0.0f, 0.0f);
}

static struct xform parse_composite(const struct crj *list) {             /* sceneloader.c:716-755 */
	if (!list) return crl_xf_identity();
	int count = crj_size(list), idx = 0;
	struct xform *tf = calloc((size_t)count + 1, sizeof(*tf));
	for (const struct crj *t = list->child; t; t = t->next) tf[idx++] = parse_transform(t);
	struct xform comp = crl_xf_identity();
	for (int i = 0; i < count; ++i) if (tf[i].type == XF_TRANSLATE) comp.A = crl_mul(&comp.A, &tf[i].A);
	for (int i = 0; i < count; ++i) if (tf[i].type <= XF_ROTATE_Z) comp.A = crl_mul(&comp.A, &tf[i].A);
	for (int i = 0; i < count; ++i) if (tf[i].type == XF_SCALE) comp.A = crl_mul(&comp.A, &tf[i].A);
	comp.Ainv = crl_inverse(&comp.A);
	comp.type = XF_COMPOSITE;
	free(tf);
	return comp;
}

/* ---- prefs + camera -------------------------------------------------------------------------------------- */
static int int_pref(const struct crj *obj, const char *key, int def, int lo, int below) {
	const struct crj *j = crj_get(obj, key);
	if (!j) return def;
	if (!crj_is_number(j)) return def;
	return j->inum >= lo ? j->inum : below;
}

static void parse_prefs(const struct crj *d, struct crs_prefs *p) {        /* sceneloader.c:190-424 */
	const int cores = (int)sysconf(_SC_NPROCESSORS_ONLN);
	*p = (struct crs_prefs){ .image_width = 1280, .image_height = 800, .sample_count = 25, .bounces = 20,
		.tile_width = 32, .tile_height = 32, .tile_order = 1 /* fromMiddle */, .thread_count = (uint32_t)cores };
	if (!d) return;
	const struct crj *threads = crj_get(d, "threads");
	if (threads && crj_is_number(threads) && threads->inum > 0) p->thread_count = (uint32_t)threads->inum;
	else if (!threads || crj_is_number(threads)) p->thread_count = (uint32_t)cores + 2;
	p->sample_count = (uint32_t)int_pref(d, "samples", 25, 1, 1);
	p->bounces = (uint32_t)int_pref(d, "bounces", 20, 0, 1);
	p->tile_width = (uint32_t)int_pref(d, "tileWidth", 32, 1, 1);
	p->tile_height = (uint32_t)int_pref(d, "tileHeight", 32, 1, 1);
	p->image_width = (uint32_t)int_pref(d, "width", 1280, 0, 640);
	p->image_height = (uint32_t)int_pref(d, "height", 800, 0, 400);
	const struct crj *order = crj_get(d, "tileOrder");
	if (crj_is_string(order)) {                                            /* enum renderOrder, tile.h:15-21 */
		if (!strcmp(order->str, "random")) p->tile_order = 4;
		else if (!strcmp(order->str, "topToBottom")) p->tile_order = 0;
		else if (!strcmp(order->str, "fromMiddle")) p->tile_order = 1;
		else if (!strcmp(order->str, "toMiddle")) p->tile_order = 2;
		else p->tile_order = 3;
	}
}

static int parse_camera(const struct crj *d, unsigned width, unsigned height, struct crs_camera *cam) {
	if (!d) { snprintf(g_err, sizeof(g_err), "scene has no \"camera\" object"); return -1; }
	float fov = 80.0f, focal = 10.0f, fstops = 0.0f;
	const struct crj *j;
	if ((j = crj_get(d, "FOV"))) {
		if (!crj_is_number(j)) goto bad;
		fov = j->num >= 0.0 ? (j->num > 180.0 ? 180.0f : (float)j->num) : 80.0f;
	}
	if ((j = crj_get(d, "focalDistance"))) {
		if (!crj_is_number(j)) goto bad;
		focal = j->num >= 0.0 ? (float)j->num : 0.0f;
	}
	if ((j = crj_get(d, "fstops"))) {
		if (!crj_is_number(j)) goto bad;
		fstops = j->num >= 0.0 ? (float)j->num : 0.0f;
	}
	struct xform comp = crl_xf_identity();
	if ((j = crj_get(d, "transforms"))) {
		if (!crj_is_array(j)) goto bad;
		comp = parse_composite(j);
	}
	/* newCamera + updateCam, src/datatypes/camera.c:16-42 */
	memset(cam, 0, sizeof(*cam));
	cam->width = (int32_t)width;
	cam->height = (int32_t)height;
	cam->focal_distance = focal;
	float aspect = (float)width / (float)height;
	cam->sensor_x = 2.0f * tanf(crl_to_radians(fov) / 2.0f);
	cam->sensor_y = cam->sensor_x / aspect;
	const float sensor_width_35mm = 0.036f;
	float focalLength = 0.5f * sensor_width_35mm / crl_to_radians(0.5f * fov);
	if (fstops != 0.0f) cam->aperture = 0.5f * (focalLength / fstops);
	const vec3 worldUp = { 0.0f, 1.0f, 0.0f };
	vec3 forward = v_norm((vec3){ 0.0f, 0.0f, 1.0f });
	vec3 right = v_cross(worldUp, forward);
	vec3 up = v_cross(forward, right);
	memcpy(cam->forward, &forward, sizeof(forward));
	memcpy(cam->right, &right, sizeof(right));
	memcpy(cam->up, &up, sizeof(up));
	memcpy(cam->A, comp.A.m, sizeof(cam->A));
	return 0;
bad:
	snprintf(g_err, sizeof(g_err), "invalid value in \"camera\"");
	return -1;
}

/* ---- node graphs ----------------------------------------------------------------------------------------- */
static int parse_texture_node(struct crl_ctx *c, const struct crj *n);

static int parse_value_node(struct crl_ctx *c, const struct crj *n) {
	if (!n) return -1;
	if (crj_is_number(n)) return crl_const_value(c, (float)n->num);
	return crl_grayscale(c, parse_texture_node(c, n));
}

static int parse_texture_node(struct crl_ctx *c, const struct crj *n) {   /* sceneloader.c:773-835 */
	if (!n) return -1;
	if (crj_is_array(n)) return crl_const_color(c, parse_color(n));
	if (crj_is_string(n)) return crl_image(c, crl_load_texture(c, n->str), 0);
	if (!crj_is_object(n)) return crl_const_color(c, crl_black);
	uint32_t options = CRS_IMG_SRGB_TRANSFORM;
	const struct crj *tr = crj_get(n, "transform");
	if (tr && !crj_is_true(tr)) options &= ~CRS_IMG_SRGB_TRANSFORM;
	if (!crj_is_true(crj_get(n, "lerp"))) options |= CRS_IMG_NO_BILINEAR;
	if (crj_get(n, "r")) return crl_const_color(c, parse_color(n));
	const struct crj *type = crj_get(n, "type");
	if (crj_is_string(type)) {
		if (!strcmp(type->str, "checkerboard")) return crl_checker(c, -1, -1, parse_value_node(c, crj_get(n, "size")));
		if (!strcmp(type->str, "blackbody")) {
			const struct crj *deg = crj_get(n, "degrees");
			return crl_blackbody(c, crl_const_value(c, crj_is_number(deg) ? (float)deg->num : 0.0f));
		}
	}
	const struct crj *path = crj_get(n, "path");
	if (crj_is_string(path)) return crl_image(c, crl_load_texture(c, path->str), options);
	fprintf(stderr, "cr_loader: unknown texture node, using black\n");
	return crl_const_color(c, crl_black);
}

static int parse_bsdf_node(struct crl_ctx *c, const struct crj *n) {      /* sceneloader.c:837-875 */
	if (!n) return -1;
	const struct crj *type = crj_get(n, "type");
	if (!crj_is_string(type)) return crl_warning_bsdf(c);
	const struct crj *color = crj_get(n, "color"), *roughness = crj_get(n, "roughness"), *strength = crj_get(n, "strength");
	int A = parse_bsdf_node(c, crj_get(n, "A"));
	int B = parse_bsdf_node(c, crj_get(n, "B"));
	const char *t = type->str;
	if (!strcmp(t, "diffuse")) return crl_diffuse(c, parse_texture_node(c, color));
	if (!strcmp(t, "metal")) { int col = parse_texture_node(c, color); return crl_metal(c, col, parse_value_node(c, roughness)); }
	if (!strcmp(t, "glass")) {
		int col = parse_texture_node(c, color), r = parse_value_node(c, roughness);
		return crl_glass(c, col, r, parse_value_node(c, crj_get(n, "IOR")));
	}
	if (!strcmp(t, "plastic")) return crl_plastic(c, parse_texture_node(c, color));
	if (!strcmp(t, "mix")) return crl_mix(c, A, B, parse_value_node(c, crj_get(n, "factor")));
	if (!strcmp(t, "add")) return crl_add(c, A, B);
	if (!strcmp(t, "transparent")) return crl_transparent(c, parse_texture_node(c, color));
	if (!strcmp(t, "emissive")) { int col = parse_texture_node(c, color); return crl_emissive(c, col, parse_value_node(c, strength)); }
	fprintf(stderr, "cr_loader: unknown bsdf node \"%s\", using the warning material\n", t);
	return crl_warning_bsdf(c);
}

/* ---- scene objects --------------------------------------------------------------------------------------- */
static void add_instance(struct crl_ctx *c, int is_mesh, int object, struct xform comp) {
	if (c->instance_count == c->instance_cap) {
		c->instance_cap = c->instance_cap ? c->instance_cap * 2 : 16;
		c->instances = realloc(c->instances, sizeof(*c->instances) * (size_t)c->instance_cap);
	}
	c->instances[c->instance_count++] = (struct crl_instance){ .composite = comp, .is_mesh = is_mesh, .object = object };
}

static void parse_ambient(struct crl_ctx *c, const struct crj *d) {        /* sceneloader.c:681-713 */
	const struct crj *offset = crj_get(d, "offset");
	int offsetValue = crj_is_number(offset) ? crl_const_value(c, crl_to_radians((float)offset->num) / 4.0f) : -1;
	const struct crj *down = crj_get(d, "down"), *up = crj_get(d, "up"), *hdr = crj_get(d, "hdr");
	if (crj_is_string(hdr)) {
		char *full = join(c->asset_path, hdr->str);
		if (file_exists(full)) {
			c->background = crl_background(c, crl_image(c, crl_load_texture(c, full), 0), -1, offsetValue);
			free(full);
			return;
		}
		free(full);
	}
	if (down && up) {
		struct crl_color dn = parse_color(down), u = parse_color(up);
		c->background = crl_background(c, crl_gradient(c, dn, u), -1, offsetValue);
		return;
	}
	c->background = crl_background(c, -1, -1, offsetValue);
}

static enum crl_bsdf_type legacy_type(const struct crj *bsdf, enum crl_bsdf_type def, int sphere) {
	if (!crj_is_string(bsdf)) return def;
	if (!strcmp(bsdf->str, "metal")) return CRL_METAL;
	if (!strcmp(bsdf->str, "glass")) return CRL_GLASS;
	if (!strcmp(bsdf->str, "plastic")) return CRL_PLASTIC;
	if (!strcmp(bsdf->str, "emissive")) return CRL_EMISSION;
	if (sphere && strcmp(bsdf->str, "lambertian")) return def;              /* spheres keep the default on unknown names */
	return CRL_LAMBERTIAN;
}

static int parse_sphere(struct crl_ctx *c, const struct crj *d) {          /* sceneloader.c:1008-1100 */
	struct crl_sphere s;
	memset(&s, 0, sizeof(s));
	s.radius = 10.0f;                                                       /* defaultSphere / defaultMaterial */
	s.material.diffuse = crl_gray;
	s.material.type = CRL_LAMBERTIAN;
	s.material.IOR = 1.0f;
	s.material.texture = s.material.specular_map = s.material.bsdf = -1;
	s.material.type = legacy_type(crj_get(d, "bsdf"), CRL_LAMBERTIAN, 1);
	const struct crj *color = crj_get(d, "color");
	if (color) {
		if (s.material.type == CRL_EMISSION) s.material.emission = parse_color(color);
		else s.material.diffuse = parse_color(color);
	}
	const struct crj *intensity = crj_get(d, "intensity");
	if (crj_is_number(intensity) && s.material.type == CRL_EMISSION)
		s.material.emission = color_coef((float)intensity->num, s.material.emission);
	s.material.roughness = num_or(crj_get(d, "roughness"), 0.0f);
	s.material.IOR = num_or(crj_get(d, "IOR"), 1.0f);
	s.radius = num_or(crj_get(d, "radius"), 10.0f);
	const int index = c->sphere_count;
	c->spheres[c->sphere_count++] = s;
	const struct crj *instances = crj_get(d, "instances");
	if (crj_is_array(instances))
		for (const struct crj *i = instances->child; i; i = i->next)
			add_instance(c, 0, index, parse_composite(crj_get(i, "transforms")));
	const struct crj *graph = crj_get(d, "material");
	if (graph) c->spheres[index].material.bsdf = parse_bsdf_node(c, graph);
	else crl_assign_bsdf(c, &c->spheres[index].material);
	return 0;
}

static int parse_mesh(struct crl_ctx *c, const struct crj *d) {            /* sceneloader.c:878-974 */
	const struct crj *fileName = crj_get(d, "fileName");
	enum crl_bsdf_type type = legacy_type(crj_get(d, "bsdf"), CRL_LAMBERTIAN, 0);
	if (!crj_is_string(fileName)) return 0;
	char *full = join(c->asset_path, fileName->str);
	struct crl_mesh mesh;
	int rc = crl_load_obj(c, full, &mesh);
	free(full);
	if (rc < 0) { snprintf(g_err, sizeof(g_err), "%s", c->err); return -1; }
	if (rc > 0) { fprintf(stderr, "cr_loader: mesh file \"%s\" not found, skipped\n", fileName->str); return 0; }
	const int index = c->mesh_count;
	c->meshes[c->mesh_count++] = mesh;
	struct crl_mesh *m = &c->meshes[index];
	const struct crj *instances = crj_get(d, "instances");
	if (crj_is_array(instances))
		for (const struct crj *i = instances->child; i; i = i->next)
			add_instance(c, 1, index, parse_composite(crj_get(i, "transforms")));
	const struct crj *materials = crj_get(d, "material");
	if (materials) {
		if (crj_is_array(materials)) {
			if (crj_size(materials) > m->material_count) {
				snprintf(g_err, sizeof(g_err), "mesh \"%s\": more material graphs than materials in its MTL", fileName->str);
				return -1;
			}
			int k = 0;
			for (const struct crj *g = materials->child; g; g = g->next) m->materials[k++].bsdf = parse_bsdf_node(c, g);
		} else {
			int node = parse_bsdf_node(c, materials);
			for (int k = 0; k < m->material_count; ++k) m->materials[k].bsdf = node;
		}
	} else {
		const struct crj *intensity = crj_get(d, "intensity"), *roughness = crj_get(d, "roughness"), *IOR = crj_get(d, "IOR");
		for (int k = 0; k < m->material_count; ++k) {
			struct crl_material *mat = &m->materials[k];
			mat->type = type;
			if (type == CRL_EMISSION && intensity) mat->emission = color_coef((float)intensity->num, mat->diffuse);
			if (type == CRL_GLASS) { if (crj_is_number(IOR)) mat->IOR = (float)IOR->num; }
			else if (type == CRL_PLASTIC) mat->IOR = (float)1.45;
			if (crj_is_number(roughness)) mat->roughness = (float)roughness->num;
			crl_assign_bsdf(c, mat);
		}
	}
	return 0;
}

/* ---- acceleration structures ----------------------------------------------------------------------------- */
struct poly_user { const struct crl_ctx *c; const struct crs_poly *polys; };

static void poly_bbox(void *user, unsigned i, bbox3 *bbox, vec3 *center) {  /* bvh.c:283-291 */
	const struct poly_user *u = user;
	const vec3 *V = (const vec3 *)u->c->vertices;
	vec3 v0 = V[u->polys[i].v[0]], v1 = V[u->polys[i].v[1]], v2 = V[u->polys[i].v[2]];
	*center = v_scale(v_add(v_add(v0, v1), v2), 1.0f / 3.0f);
	bbox->min = v_min(v0, v_min(v1, v2));
	bbox->max = v_max(v0, v_max(v1, v2));
}

static void instance_bbox(void *user, unsigned i, bbox3 *bbox, vec3 *center) {
	struct crl_ctx *c = user;
	const struct crl_instance *in = &c->instances[i];
	if (in->is_mesh) {                                                      /* instance.c:221-230 */
		struct crl_mesh *m = &c->meshes[in->object];
		const float *b = m->bvh_nodes[0].bounds;
		*bbox = (bbox3){ { b[0], b[2], b[4] }, { b[1], b[3], b[5] } };
		crl_transform_bbox(bbox, &in->composite.A);
		*center = bbox_center(bbox);
		m->ray_offset = bbox_ray_offset(*bbox);
	} else {                                                                /* instance.c:94-110 */
		struct crl_sphere *s = &c->spheres[in->object];
		*center = crl_point((vec3){ 0.0f, 0.0f, 0.0f }, &in->composite.A);
		bbox->min = (vec3){ -s->radius, -s->radius, -s->radius };
		bbox->max = (vec3){ s->radius, s->radius, s->radius };
		const enum xf_type t = in->composite.type;
		if (!(t <= XF_ROTATE_Z) && t != XF_TRANSLATE) crl_transform_bbox(bbox, &in->composite.A);
		else { bbox->min = v_add(bbox->min, *center); bbox->max = v_add(bbox->max, *center); }
		s->ray_offset = bbox_ray_offset(*bbox);
	}
}

/* ---- flattening (order of oracle/ref_harness.c flatten()) --------------------------------------------------- */
struct flat {
	const struct crl_ctx *c;
	int *node_map, *tex_map;       /* loader handle -> flat index, -1 = not yet emitted */
	struct crs_node *nodes; int node_count;
	int *tex_order; int tex_count;
};

static int flat_node(struct flat *f, int handle) {
	if (handle < 0) return -1;
	if (f->node_map[handle] >= 0) return f->node_map[handle];
	const struct crl_node *n = &f->c->nodes[handle];
	const int idx = f->node_count++;
	f->node_map[handle] = idx;
	int in[3];
	for (int k = 0; k < 3; ++k) in[k] = flat_node(f, n->in[k]);
	struct crs_node *d = &f->nodes[idx];
	memset(d, 0, sizeof(*d));
	d->kind = n->kind;
	memcpy(d->in, in, sizeof(in));
	memcpy(d->f, n->f, sizeof(d->f));
	d->tex = -1;
	if (n->tex >= 0) {
		if (f->tex_map[n->tex] < 0) { f->tex_map[n->tex] = f->tex_count; f->tex_order[f->tex_count++] = n->tex; }
		d->tex = f->tex_map[n->tex];
	}
	d->options = n->options;
	return idx;
}

static void flat_material(struct flat *f, struct crs_material *d, const struct crl_material *m) {
	d->emission[0] = m->emission.r; d->emission[1] = m->emission.g; d->emission[2] = m->emission.b; d->emission[3] = m->emission.a;
	d->IOR = m->IOR;
	d->bsdf = flat_node(f, m->bsdf);
}

static size_t align16(size_t n) { return (n + 15u) & ~(size_t)15u; }

static int flatten(struct crl_ctx *c, const struct crs_prefs *prefs, const struct crs_camera *cam,
                   struct crs_bvh_node *top_nodes, uint32_t top_count, int32_t *top_prims, struct crs_scene *s) {
	struct flat f = { .c = c };
	f.node_map = malloc(sizeof(int) * ((size_t)c->node_count + 1));
	f.tex_map = malloc(sizeof(int) * ((size_t)c->texture_count + 1));
	f.tex_order = malloc(sizeof(int) * ((size_t)c->texture_count + 1));
	f.nodes = calloc((size_t)c->node_count + 1, sizeof(*f.nodes));
	for (int i = 0; i < c->node_count; ++i) f.node_map[i] = -1;
	for (int i = 0; i < c->texture_count; ++i) f.tex_map[i] = -1;

	uint32_t matCount = (uint32_t)c->sphere_count, polyCount = 0, nodeTotal = top_count, primTotal = (uint32_t)c->instance_count;
	for (int m = 0; m < c->mesh_count; ++m) {
		matCount += (uint32_t)c->meshes[m].material_count;
		polyCount += (uint32_t)c->meshes[m].poly_count;
		nodeTotal += c->meshes[m].bvh_node_count;
		primTotal += (uint32_t)c->meshes[m].poly_count;
	}
	struct crs_material *materials = calloc((size_t)matCount + 1, sizeof(*materials));
	uint32_t mat = 0;
	for (int m = 0; m < c->mesh_count; ++m)
		for (int k = 0; k < c->meshes[m].material_count; ++k) flat_material(&f, &materials[mat++], &c->meshes[m].materials[k]);
	const uint32_t sphere_mat0 = mat;
	for (int i = 0; i < c->sphere_count; ++i) flat_material(&f, &materials[mat++], &c->spheres[i].material);
	const int background = flat_node(&f, c->background);

	uint64_t texBytes = 0;
	for (int i = 0; i < f.tex_count; ++i) {
		const struct cr_image *t = &c->textures[f.tex_order[i]];
		texBytes += align16((size_t)t->width * t->height * t->channels * (t->is_float ? 4u : 1u));
	}

	/* one backing block, arrays 16-byte aligned (freed by crscene_free through `owner`) */
	size_t sizes[14] = {
		sizeof(struct crs_instance) * (size_t)c->instance_count, sizeof(struct crs_sphere) * (size_t)c->sphere_count,
		sizeof(struct crs_mesh) * (size_t)c->mesh_count, sizeof(struct crs_material) * matCount,
		sizeof(struct crs_node) * (size_t)f.node_count, sizeof(struct crs_texture) * (size_t)f.tex_count,
		sizeof(struct crs_bvh) * ((size_t)c->mesh_count + 1), sizeof(struct crs_bvh_node) * nodeTotal,
		sizeof(int32_t) * primTotal, sizeof(struct crs_poly) * polyCount,
		sizeof(float) * 3 * (size_t)c->vertex_count, sizeof(float) * 3 * (size_t)c->normal_count,
		sizeof(float) * 2 * (size_t)c->texcoord_count, (size_t)texBytes };
	size_t total = 16;
	for (int i = 0; i < 14; ++i) total += align16(sizes[i]) + 16;
	uint8_t *block = calloc(total, 1);
	if (!block) { snprintf(g_err, sizeof(g_err), "out of memory"); return -1; }
	uint8_t *cursor = block;
	void *arr[14];
	for (int i = 0; i < 14; ++i) { arr[i] = cursor; cursor += align16(sizes[i]) + 16; }

	memset(s, 0, sizeof(*s));
	s->owner = block;
	s->prefs = *prefs;
	s->camera = *cam;
	s->instances = arr[0]; s->spheres = arr[1]; s->meshes = arr[2]; s->materials = arr[3]; s->nodes = arr[4];
	s->textures = arr[5]; s->bvhs = arr[6]; s->bvh_nodes = arr[7]; s->prim_indices = arr[8]; s->polys = arr[9];
	s->vertices = arr[10]; s->normals = arr[11]; s->texcoords = arr[12]; s->texdata = arr[13];
	s->instance_count = (uint32_t)c->instance_count; s->sphere_count = (uint32_t)c->sphere_count;
	s->mesh_count = (uint32_t)c->mesh_count; s->material_count = matCount; s->node_count = (uint32_t)f.node_count;
	s->texture_count = (uint32_t)f.tex_count; s->bvh_count = (uint32_t)c->mesh_count + 1;
	s->bvh_node_count = nodeTotal; s->prim_index_count = primTotal; s->poly_count = polyCount;
	s->vertex_count = (uint32_t)c->vertex_count; s->normal_count = (uint32_t)c->normal_count;
	s->texcoord_count = (uint32_t)c->texcoord_count; s->texdata_bytes = texBytes;
	s->background = background;
	s->top_bvh = (uint32_t)c->mesh_count;

	memcpy(s->materials, materials, sizeof(*materials) * matCount);
	memcpy(s->nodes, f.nodes, sizeof(struct crs_node) * (size_t)f.node_count);
	uint32_t poly = 0, node = 0, prim = 0;
	mat = 0;
	for (int m = 0; m < c->mesh_count; ++m) {
		const struct crl_mesh *src = &c->meshes[m];
		s->meshes[m] = (struct crs_mesh){ .poly_offset = poly, .poly_count = (uint32_t)src->poly_count, .material_offset = mat,
			.material_count = (uint32_t)src->material_count, .texcoord_count = (uint32_t)src->texcoord_count,
			.bvh = (uint32_t)m, .ray_offset = src->ray_offset };
		s->bvhs[m] = (struct crs_bvh){ node, src->bvh_node_count, prim, (uint32_t)src->poly_count };
		if (src->bvh_node_count) memcpy(s->bvh_nodes + node, src->bvh_nodes, sizeof(struct crs_bvh_node) * src->bvh_node_count);
		if (src->poly_count) {
			memcpy(s->prim_indices + prim, src->bvh_prims, sizeof(int32_t) * (size_t)src->poly_count);
			memcpy(s->polys + poly, src->polys, sizeof(struct crs_poly) * (size_t)src->poly_count);
		}
		poly += (uint32_t)src->poly_count; prim += (uint32_t)src->poly_count; node += src->bvh_node_count;
		mat += (uint32_t)src->material_count;
	}
	for (int i = 0; i < c->sphere_count; ++i)
		s->spheres[i] = (struct crs_sphere){ .radius = c->spheres[i].radius, .ray_offset = c->spheres[i].ray_offset, .material = sphere_mat0 + (uint32_t)i };
	for (int i = 0; i < c->instance_count; ++i) {
		struct crs_instance *d = &s->instances[i];
		memcpy(d->A, c->instances[i].composite.A.m, sizeof(d->A));
		memcpy(d->Ainv, c->instances[i].composite.Ainv.m, sizeof(d->Ainv));
		d->kind = c->instances[i].is_mesh ? CRS_INST_MESH : CRS_INST_SPHERE;
		d->object = (uint32_t)c->instances[i].object;
	}
	s->bvhs[c->mesh_count] = (struct crs_bvh){ node, top_count, prim, (uint32_t)c->instance_count };
	if (top_count) memcpy(s->bvh_nodes + node, top_nodes, sizeof(struct crs_bvh_node) * top_count);
	if (c->instance_count) memcpy(s->prim_indices + prim, top_prims, sizeof(int32_t) * (size_t)c->instance_count);
	if (c->vertex_count) memcpy(s->vertices, c->vertices, sizeof(float) * 3 * (size_t)c->vertex_count);
	if (c->normal_count) memcpy(s->normals, c->normals, sizeof(float) * 3 * (size_t)c->normal_count);
	if (c->texcoord_count) memcpy(s->texcoords, c->texcoords, sizeof(float) * 2 * (size_t)c->texcoord_count);
	uint64_t off = 0;
	for (int i = 0; i < f.tex_count; ++i) {
		const struct cr_image *t = &c->textures[f.tex_order[i]];
		size_t bytes = (size_t)t->width * t->height * t->channels * (t->is_float ? 4u : 1u);
		s->textures[i] = (struct crs_texture){ .width = t->width, .height = t->height, .channels = t->channels,
			.is_float = (uint32_t)t->is_float, .has_alpha = (!t->is_float && t->channels > 3) ? 1u : 0u, .data_offset = off };
		memcpy(s->texdata + off, t->data, bytes);
		off += align16(bytes);
	}
	free(materials); free(f.node_map); free(f.tex_map); free(f.tex_order); free(f.nodes);
	return 0;
}

/* ---- entry point ------------------------------------------------------------------------------------------ */
static void ctx_free(struct crl_ctx *c) {
	crl_textures_join(c);                                  /* error paths: no decode thread may outlive the context */
	free(c->tex_jobs);
	for (int m = 0; m < c->mesh_count; ++m) {
		struct crl_mesh *mesh = &c->meshes[m];
		for (int k = 0; k < mesh->material_count; ++k) free(mesh->materials[k].name);
		free(mesh->materials); free(mesh->polys); free(mesh->bvh_nodes); free(mesh->bvh_prims);
	}
	for (int i = 0; i < c->texture_count; ++i) free(c->textures[i].data);
	free(c->textures); free(c->meshes); free(c->spheres); free(c->instances); free(c->nodes);
	free(c->vertices); free(c->normals); free(c->texcoords); free(c->asset_path);
}

static int load_text(struct crs_scene *out, const char *text, const char *asset_path, const char *what, struct crloader_output *output);
static int load_text_mode(struct crs_scene *out, const char *text, const char *asset_path, const char *what, struct crloader_output *output, int async);

int crloader_load_json(struct crs_scene *out, const char *json_path) {
	g_err[0] = '\0';
	if (!out || !json_path) { snprintf(g_err, sizeof(g_err), "null argument"); return -1; }
	char *text = slurp(json_path);
	if (!text) { snprintf(g_err, sizeof(g_err), "cannot read %s", json_path); return -2; }
	char *copy = strdup(json_path);
	char *assets = join(dirname(copy), "/");                 /* c-ray.c:254-256 */
	int rc = load_text(out, text, assets, json_path, NULL);
	free(assets); free(copy); free(text);
	return rc;
}

int crloader_load_json_buf(struct crs_scene *out, const char *json_text, const char *asset_path, struct crloader_output *output) {
	g_err[0] = '\0';
	if (!out || !json_text) { snprintf(g_err, sizeof(g_err), "null argument"); return -1; }
	return load_text(out, json_text, asset_path ? asset_path : "./", "<buffer>", output);
}

static void parse_output(const struct crj *d, struct crloader_output *o) {   /* sceneloader.c:341-424, defaults :190-208 */
	snprintf(o->file_path, sizeof(o->file_path), "./");
	snprintf(o->file_name, sizeof(o->file_name), "rendered");
	o->count = 0;
	o->type = 1;
	if (!d) return;
	const struct crj *j;
	if (crj_is_string(j = crj_get(d, "outputFilePath"))) snprintf(o->file_path, sizeof(o->file_path), "%s", j->str);
	if (crj_is_string(j = crj_get(d, "outputFileName"))) snprintf(o->file_name, sizeof(o->file_name), "%s", j->str);
	if (crj_is_number(j = crj_get(d, "count"))) o->count = j->inum >= 0 ? j->inum : 0;
	if (crj_is_string(j = crj_get(d, "fileType"))) o->type = !strcmp(j->str, "bmp") ? 0 : 1;
}

static int load_text(struct crs_scene *out, const char *text, const char *asset_path, const char *what, struct crloader_output *output) {
	const int async = crl_thread_count() > 1 && !getenv("CRLOADER_SYNC_TEXTURES");
	int rc = load_text_mode(out, text, asset_path, what, output, async);
	if (rc == -100) rc = load_text_mode(out, text, asset_path, what, output, 0);   /* a background decode failed late: redo in order */
	return rc;
}

static int load_text_mode(struct crs_scene *out, const char *text, const char *asset_path, const char *what, struct crloader_output *output, int async) {
	struct crj *json = crj_parse(text);
	if (!json) { snprintf(g_err, sizeof(g_err), "%s: JSON syntax error", what); return -3; }
	if (output) parse_output(crj_get(json, "renderer"), output);

	struct crl_ctx ctx;
	memset(&ctx, 0, sizeof(ctx));
	ctx.background = -1;
	ctx.asset_path = strdup(asset_path);
	ctx.async_textures = async;
	struct crs_prefs prefs;
	struct crs_camera cam;
	struct crs_bvh_node *top_nodes = NULL;
	int32_t *top_prims = NULL;
	uint32_t top_count = 0;
	int rc = -4;

	parse_prefs(crj_get(json, "renderer"), &prefs);
	if (!prefs.image_width || !prefs.image_height) { snprintf(g_err, sizeof(g_err), "image size is zero"); goto done; }
	if (parse_camera(crj_get(json, "camera"), prefs.image_width, prefs.image_height, &cam)) goto done;

	const struct crj *scene = crj_get(json, "scene");
	parse_ambient(&ctx, crj_get(scene, "ambientColor"));
	const struct crj *prims = crj_get(scene, "primitives");
	if (crj_is_array(prims)) {
		ctx.spheres = calloc((size_t)crj_size(prims) + 1, sizeof(*ctx.spheres));
		for (const struct crj *p = prims->child; p; p = p->next)
			if (str_eq(crj_get(p, "type"), "sphere")) parse_sphere(&ctx, p);
	}
	const struct crj *meshes = crj_get(scene, "meshes");
	if (crj_is_array(meshes)) {
		ctx.meshes = calloc((size_t)crj_size(meshes) + 1, sizeof(*ctx.meshes));
		for (const struct crj *m = meshes->child; m; m = m->next) if (parse_mesh(&ctx, m)) goto done;
	}

	/* bottom-level BVHs, then the top level (whose bbox callbacks also set every ray offset) */
	for (int m = 0; m < ctx.mesh_count; ++m) {
		struct crl_mesh *mesh = &ctx.meshes[m];
		for (int p = 0; p < mesh->poly_count; ++p)
			for (int k = 0; k < 3; ++k)
				if (mesh->polys[p].v[k] < 0 || mesh->polys[p].v[k] >= ctx.vertex_count) {
					snprintf(g_err, sizeof(g_err), "mesh %d: face %d refers to a vertex outside the file", m, p);
					goto done;
				}
		struct poly_user u = { &ctx, mesh->polys };
		if (crl_build_bvh(&u, poly_bbox, (unsigned)mesh->poly_count, &mesh->bvh_nodes, &mesh->bvh_node_count, &mesh->bvh_prims)) {
			snprintf(g_err, sizeof(g_err), "out of memory"); goto done;
		}
	}
	for (int i = 0; i < ctx.instance_count; ++i)
		if (ctx.instances[i].is_mesh && ctx.meshes[ctx.instances[i].object].bvh_node_count == 0) {
			snprintf(g_err, sizeof(g_err), "instance %d refers to a mesh without polygons", i);
			goto done;
		}
	if (crl_build_bvh(&ctx, instance_bbox, (unsigned)ctx.instance_count, &top_nodes, &top_count, &top_prims)) {
		snprintf(g_err, sizeof(g_err), "out of memory"); goto done;
	}

	/* renderer.c / scene.c:206-210: never more workers than tiles */
	{
		uint32_t tx = (prefs.image_width + prefs.tile_width - 1) / prefs.tile_width;
		uint32_t ty = (prefs.image_height + prefs.tile_height - 1) / prefs.tile_height;
		if (tx * ty < prefs.thread_count) prefs.thread_count = tx * ty;
	}
	crl_textures_join(&ctx);
	if (ctx.async_failed) { rc = -100; goto done; }
	rc = flatten(&ctx, &prefs, &cam, top_nodes, top_count, top_prims, out) ? -5 : 0;
done:
	free(top_nodes); free(top_prims);
	ctx_free(&ctx);
	crj_free(json);
	return rc;
}
