/*
 * crgpu_bvh_build.cuh — the device SAH builder (crgpu_bvh_build.cu) as the scene-edit path uses it: on the scene's stream, from
 * device-resident inputs, into caller-owned scratch, with a BVH (the top level or a mesh's) laid out as crgpu_api.cu build_pairs lays
 * out an uploaded one.
 */
#pragma once
#include <cuda_runtime.h>
#include "crgpu_scene.cuh"

/* Declared weak: a program that links the upload path without the builder (tests/stub/create_harness.c, which hashes the slab)
 * still links; libcrgpu.so always defines them. */
#define CRG_WEAK __attribute__((weak))

/* bytes of device scratch crg_bvh_build_pairs needs for n primitives (reusable for any later build of at most n) */
CRG_WEAK size_t crg_bvh_scratch_bytes(uint32_t n);

struct CrgBuildResult {
	uint32_t node_count;            /* reference nodeCount (bvh.c) */
	uint32_t pairs;                 /* internal nodes = pair nodes written (0 when node_count <= 1) */
	uint32_t levels;                /* BFS levels holding internal nodes (the deepest internal node is at depth levels - 1) */
	uint32_t root_first, root_count;/* node_count == 1: the root leaf's range */
	float    bounds[6];             /* root bounds as stored (minx,maxx,miny,maxy,minz,maxz) */
};

/* The tree crgpu_bvh_build builds over n primitives (bb: n x 6 min xyz max xyz, ctr: n x 3, both device), enqueued on st.  Writes
 * the internal nodes as PairNodes in build_pairs' BFS order with local refs into pairs_out (room for max(1, n - 1)) and the
 * primitive order into prims_out (n, device); returns when both are written (st is synchronised). */
CRG_WEAK int crg_bvh_build_pairs(const float *bb, const float *ctr, uint32_t n, void *scratch, cudaStream_t st, PairNode *pairs_out, int32_t *prims_out,
					  CrgBuildResult *out);

/* instance_bbox of the scene loader (host/loader/cr_sceneload.c) for n edited instances: each DevInstance takes A / Ainv from inst
 * (inst == NULL: keeps its own, as a mesh edit does), bb / ctr (device, n x 6 and n x 3) receive the top-level build's inputs and every instance the ray offset of the last instance of
 * its object (last[i]).  bvh_root: 6 floats per BVH, the root bounds of each mesh BVH as stored. */
CRG_WEAK void crg_launch_instance_boxes(const crs_instance *inst, DevInstance *insts, const float *bvh_root, const uint32_t *last, uint32_t n,
							   float *bb, float *ctr, float *offs, cudaStream_t st);

/* the top level's item records (DevTopItem) for the edited instances: item i describes instance prims[i] of insts (device, n each) */
CRG_WEAK void crg_launch_top_items(const int32_t *prims, const DevInstance *insts, const DevBvh *bvhs, uint32_t n, DevTopItem *items, cudaStream_t st);

/* poly_bbox of the scene loader (host/loader/cr_sceneload.c <- bvh.c:283-291) for the n polys of one mesh: bb (n x 6) and ctr (n x 3),
 * the bottom-level build's inputs.  Vertex v of a poly is verts[3 * (v - vbase)]: the caller uploads the range the mesh indexes. */
CRG_WEAK void crg_launch_poly_boxes(const crs_poly *polys, const float *verts, uint32_t vbase, uint32_t n, float *bb, float *ctr, cudaStream_t st);

/* One mesh's slot-ordered and poly-ordered records, as crgpu_prepare packs them (steps 2 and 3 and the shading keys), from its polys
 * (device, n) and the primitive order prims of its new BVH.  Slot i takes poly prims[i]: tris[i], slot_poly[i] = poly_offset +
 * prims[i], keys[i]; spolys[j] is the record of poly j.  verts / normals / uvs hold the ranges from vbase / nbase / tbase the polys
 * index (crgpu_api.cu has checked every index). */
struct CrgMeshRepack {
	const crs_poly *polys;
	const float *verts, *normals, *uvs;
	uint32_t vbase, nbase, tbase;
	uint32_t n, poly_offset, material_offset, texcoord_count;
};
CRG_WEAK void crg_launch_mesh_repack(const CrgMeshRepack &m, const int32_t *prims, PackedTri *tris, uint32_t *slot_poly, uint8_t *keys,
                                     ShadePoly *spolys, cudaStream_t st);

/* The builder's inclusive prefix sum of n 64-bit words (the two 32-bit halves summed independently: each must stay below 2^32), for
 * n <= 2^30, enqueued on st.  `in` may be `out`.  sums holds ceil(n / 1024) words and sums2 ceil(n / 2^20) (at most 1024) words of
 * scratch.  Returns the number of kernels it launched. */
CRG_WEAK int crg_scan64(const unsigned long long *in, unsigned long long *out, unsigned long long *sums, unsigned long long *sums2, uint32_t n,
                        cudaStream_t st);
