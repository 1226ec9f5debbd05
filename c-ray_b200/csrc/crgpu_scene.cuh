/*
 * crgpu_scene.cuh — device-side scene layout (HBM) for the H100 hot path.
 *
 * Built once per scene by crgpu_scene_create() from the flat description (include/crscene.h).
 * The reference layout is pointer-linked AoS (struct bvhNode 32 B bvh.c:37-42, struct poly 40 B of
 * indices poly.h:11-18 into global vertex arrays, struct instance 160 B instance.h:23-28).  Here:
 *
 *   PairNode  64 B, 64-B aligned: BOTH children of one internal node (bounds + refs), because the
 *             traversal always fetches and tests the two children together (bvh.c:392-398).  One
 *             LDG.128 x4 per step instead of two dependent 32-B fetches; internal nodes are renumbered
 *             in BFS order so the top of each tree is one contiguous range (staged into shared memory
 *             by TMA bulk copies in the traversal kernel).
 *   PackedTri 48 B, 16-B aligned, in LEAF ORDER (indexed by primIndices slot, not by poly): v0, e1, e2
 *             and n = e1 x e2 precomputed with the reference's exact fp32 operations (poly.c:20-22), so
 *             a leaf's triangles are contiguous and the Möller–Trumbore test needs no index chasing.
 *   ShadePoly 80 B per poly: pre-gathered vertex normals / texcoords / material for the shade kernel.
 *   Instance  128 B: Ainv and A (3x4 rows each), kind, object parameters.
 */
#pragma once
/* limits of the device node interpreter (crgpu_shade.cuh), enforced at upload (crgpu_api.cu check_bsdf) */
#define CRG_NODE_DEPTH 3      /* color->value->color nesting of the hot interpreter (NodeEval: the node kinds JSON scenes contain) */
#define CRG_XNODE_DEPTH 8     /* edges below the first node of a kind only the complete interpreter knows (NodeX: SURVEY 8 f4) */
#define CRG_ADD_STACK 4       /* operand stack of nested ADD bsdfs */
#include <stdint.h>
#include <string.h>
#include "../../include/crscene.h"

#define CRG_LEAF_BIT 0x80000000u
#define CRG_MAX_STACK 64            /* MAX_BVH_DEPTH, bvh.c:32 */
#define CRG_STAGE_PAIRS 1024         /* 64 KB of shared memory per block for the staged top-of-tree nodes */

struct __align__(64) PairNode {
	float lb[6];                    /* left child: minx,maxx,miny,maxy,minz,maxz */
	float rb[6];                    /* right child */
	uint32_t lref, rref;            /* internal child: its pair index; leaf child: first prim slot (local to the BVH) */
	uint32_t lmeta, rmeta;          /* CRG_LEAF_BIT | primCount for leaves, 0 for internal children */
};

struct __align__(16) PackedTri {
	float v0[3], e1[3], e2[3], n[3];
};

struct __align__(16) ShadePoly {
	float n0[3], n1[3], n2[3];      /* vertex normals (n0 = geometric normal when !has_normals) */
	float t0[2], t1[2], t2[2];      /* texture coordinates */
	uint32_t material;              /* global material index */
	uint32_t flags;                 /* bit0 has_normals, bit1 has_uv */
	uint32_t pad[3];
};

struct DevBvh {
	uint32_t pair_offset;           /* into pairs[] */
	uint32_t pair_end;              /* one past this BVH's last pair node */
	uint32_t node_count;            /* reference nodeCount (0, 1 or >1 select the code path, bvh.c:362-387) */
	uint32_t slot_offset;           /* into tris[] / slot_poly[] (mesh) or top_items[] (top level) */
	uint32_t root_first, root_count;/* when node_count == 1: the root is a leaf */
	float    root_bounds[6];
	uint32_t stage_base;            /* the first stage_count pair nodes (BFS order = top of the tree) of this BVH are also */
	uint32_t stage_count;           /* in the staging image at [stage_base, stage_base+stage_count) — see DevScene.stage_img */
	uint32_t pad;
};

struct __align__(16) DevInstance {
	float Ainv[12];
	float A[12];
	uint32_t kind;                  /* CRS_INST_SPHERE / CRS_INST_MESH */
	uint32_t bvh;                   /* mesh: index into bvhs[] */
	float    ray_offset;
	float    radius;                /* sphere */
	uint32_t material;              /* sphere: global material index */
	uint32_t pad[3];
};

/* One top-level leaf item (DevScene::top_items, indexed like the top level's primIndices: top.slot_offset + item): what the
 * traversal's instance step reads, in one 64-byte record it fetches with four 16-byte loads instead of three dependent lookups
 * (primIndices, then the instance, then its mesh's DevBvh).  Only a mesh whose BVH has at most one node, or staged nodes, still
 * sends the step to bvhs[instances[i].bvh].  crgpu_prepare builds the records from the uploaded scene, an instance edit
 * (crgpu_scene_set_instances) rebuilds them on the device with k_top_items; both call crg_top_item. */
#define CRG_ITEM_MESH  0x80000000u  /* bits of DevTopItem::inst above the instance index */
#define CRG_ITEM_BVH   0x40000000u  /* a mesh whose BVH has node_count <= 1 or stage_count > 0 */
#define CRG_ITEM_INDEX 0x3fffffffu
struct __align__(16) DevTopItem {
	float Ainv[12];                 /* the instance's */
	uint32_t inst;                  /* instance index | CRG_ITEM_MESH | CRG_ITEM_BVH */
	float    ray_offset;            /* the instance's */
	uint32_t shape;                 /* sphere: radius (float bits); mesh: its BVH's pair_offset */
	uint32_t slot_offset;           /* mesh: its BVH's slot_offset; sphere: 0 */
};
static_assert(sizeof(DevTopItem) == 64, "DevTopItem is one 64-byte record");

__host__ __device__ inline DevTopItem crg_top_item(const DevInstance &in, const DevBvh *bvhs, uint32_t inst) {
	DevTopItem t;
	for (int k = 0; k < 12; ++k) t.Ainv[k] = in.Ainv[k];
	t.inst = inst;
	t.ray_offset = in.ray_offset;
	t.shape = 0u;
	t.slot_offset = 0u;
	if (in.kind == CRS_INST_MESH) {
		const DevBvh &b = bvhs[in.bvh];
		t.inst |= CRG_ITEM_MESH | (b.node_count <= 1u || b.stage_count ? CRG_ITEM_BVH : 0u);
		t.shape = b.pair_offset;
		t.slot_offset = b.slot_offset;
	} else {
		memcpy(&t.shape, &in.radius, sizeof t.shape);
	}
	return t;
}

struct DevMaterial {
	float emission[3];
	float IOR;
	int32_t bsdf;
	uint32_t flags;                 /* bit0: graph reads uv (image / checker nodes); bit1: emission != 0 */
	uint32_t pad[2];
};

/* A "flat" material, folded at upload (crgpu_api.cu fold_flat): a leaf bsdf whose inputs are constants or one image node,
 * optionally under the loader's legacy wrapper MIX(TRANSPARENT(c0), leaf, ALPHA(c)).  The flat hit launch of K3 samples it with
 * a call-free switch instead of the node interpreter; the fields are bit copies of what the interpreter would read. */
#define CRG_FLAT_NONE     0u        /* generic: the interpreter shades it */
#define CRG_FLAT_DIFFUSE  1u
#define CRG_FLAT_METAL    2u
#define CRG_FLAT_GLASS    3u
#define CRG_FLAT_EMISSIVE 4u
#define CRG_FLAT_PLASTIC  5u        /* over a diffuse: col is the diffuse's colour, rough the plastic's in[1].r */
#define CRG_FLAT_WRAPPED  1u        /* flags: the legacy alpha wrapper */
#define CRG_FLAT_ALPHA_IMG 2u       /* flags: the wrapper's alpha is an image node (else the constant alpha) */
#define CRG_FLAT_COL_IMG  4u        /* flags: the leaf colour is an image node (else col) */
struct __align__(16) DevFlat {
	uint32_t kind, flags;
	int32_t  col_tex;  uint32_t col_opt;       /* image colour: crs_node.tex / .options */
	int32_t  alpha_tex; uint32_t alpha_opt;    /* image alpha */
	float    col[4];                           /* constant leaf colour (f[0..3]) */
	float    c0[4];                            /* the wrapper's transparent colour */
	float    alpha;                            /* constant alpha (f[3] of the wrapper's alpha colour) */
	float    rough, ior, strength;             /* value inputs (f[0]); plastic: rough = f[0] of its roughness colour */
};

/* A folded background (crgpu_api.cu fold_background): BACKGROUND(colour, strength, offset) whose colour is a constant, an image
 * or a gradient and whose strength and offset are value constants — every background the JSON loader builds.  The miss launch
 * of K3 samples it inline (cr_sample_flat_bg) instead of calling the node interpreter; the fields are bit copies of the node
 * fields cr_sample_background reads. */
#define CRG_BG_NONE     0u          /* generic: the interpreter samples it */
#define CRG_BG_CONSTANT 1u
#define CRG_BG_IMAGE    2u
#define CRG_BG_GRADIENT 3u
struct DevFlatBg {
	uint32_t kind;
	int32_t  tex;  uint32_t opt;               /* image colour: crs_node.tex / .options */
	float    strength, offset;                 /* f[0] of the value constants */
	float    f[8];                             /* the colour node's f: constant f[0..3], gradient down f[0..3] / up f[4..7] */
};

struct DevTexture {
	uint32_t width, height, channels, is_float, has_alpha;
	uint32_t wmask, hmask;          /* width-1 / height-1 when that dimension is a power of two, else 0 (x % W == x & (W-1), also for the
	                                   2^64-wrapped negative coordinates of texture.c:34-35) */
	uint32_t pad;
	const uint8_t *data;
};

struct DevCamera {
	float sensor_x, sensor_y, aperture, focal_distance;
	float forward[3], right[3], up[3];
	int32_t width, height;
	float A[12];
};

struct DevScene {
	DevCamera cam;
	uint32_t image_width, image_height, sample_count, bounces;
	int32_t  background;
	uint32_t instance_count;
	DevBvh   top;
	const PairNode   *pairs;
	const PackedTri  *tris;
	const uint32_t   *slot_poly;    /* prim slot -> global poly index */
	const uint8_t    *slot_key;     /* prim slot -> shading key min(material + 1, 255) of its poly (K2's write-back: one load per hit) */
	const uint8_t    *inst_key;     /* instance -> shading key of a sphere instance (0 for meshes) */
	const ShadePoly  *spolys;
	const DevTopItem *top_items;    /* one record per top-level primIndices entry (DevTopItem) */
	const DevBvh     *bvhs;
	const DevInstance*instances;
	const DevMaterial*materials;
	const DevFlat    *flat;         /* [material] folded flat record (kind CRG_FLAT_NONE: generic) */
	const uint8_t    *key_order;    /* [256] K4's bucket order: the miss key, the keys of flat materials, then the generic keys */
	uint32_t          flat_keys;    /* number of flat keys (they take ranks 1..flat_keys of key_order) */
	DevFlatBg         bg;           /* folded background (kind CRG_BG_NONE: the interpreter samples nodes[background]) */
	const crs_node   *nodes;
	const DevTexture *textures;
	const PairNode   *stage_img;    /* top-of-tree pair nodes of every BVH, contiguous: K2 copies it into shared memory with one
	                                   TMA bulk copy (cp.async.bulk) per block; stage_pairs = number of nodes in it */
	uint32_t          stage_pairs;
	const float      *u8_to_unit;   /* [256]: (float)i / 255.0f, the byte→float division of texture.c:48-60 done once */
	/* top-level BVH bounds: lower corner and 1/extent.  Only dir mode 3 (K4b) bins origins with them; in a scene whose box is
	 * stretched by far geometry (hdr.json's emissive spheres, ~1500 units out) every secondary origin lands in one cell, which
	 * is why mode 4 bins inside the bounds of the origins themselves (WaveBuffers::box) */
	float             world_lo[3], world_inv[3];
};
