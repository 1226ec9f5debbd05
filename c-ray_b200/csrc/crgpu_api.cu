/*
 * crgpu_api.cu — C ABI of libcrgpu.so (include/crgpu.h): scene upload, the per-tile wavefront driver,
 * framebuffer access.  Host code here only lays data out in HBM and launches kernels; all arithmetic
 * of the hot path is in the kernels (crgpu_kernels.cuh).  No CPU fallback exists.
 */
#include "../../include/crgpu.h"
#include "crgpu_wave.cuh"
#include "crgpu_scene.cuh"
#include "crgpu_bvh_build.cuh"

#define CRG_HITKAT_BYTES 160
#define CRG_TAIL_FROM 6      /* first bounce at which the tail kernel may take over (it only does when <= 16384 rays are left) */

#include <cstdio>
#include <cmath>
#include <cstdlib>
#include <cstring>
#include <cstdarg>
#include <vector>
#include <algorithm>
#include <queue>
#include <deque>
#include <utility>
#include <thread>
#include <mutex>

static thread_local char g_err[512] = "";

static int fail(int code, const char *fmt, ...) {
	va_list vl;
	va_start(vl, fmt);
	vsnprintf(g_err, sizeof g_err, fmt, vl);
	va_end(vl);
	return code;
}
/* the same for the other translation units of libcrgpu.so (crgpu_bvh_build.cu) */
int crg_fail(int code, const char *fmt, ...) {
	va_list vl;
	va_start(vl, fmt);
	vsnprintf(g_err, sizeof g_err, fmt, vl);
	va_end(vl);
	return code;
}
#define CU(call) do { cudaError_t e_ = (call); if (e_ != cudaSuccess) return fail(CRGPU_ERR_CUDA, "%s: %s (%s:%d)", #call, cudaGetErrorString(e_), __FILE__, __LINE__); } while (0)

extern "C" const char *crgpu_last_error(void) { return g_err; }

extern "C" int crgpu_device_count(int *n) {
	if (!n) return fail(CRGPU_ERR_BAD_ARGUMENT, "n is NULL");
	int c = 0;
	cudaError_t e = cudaGetDeviceCount(&c);
	if (e != cudaSuccess || c < 1) { *n = 0; return fail(CRGPU_ERR_NO_DEVICE, "no CUDA device: %s", cudaGetErrorString(e)); }
	*n = c;
	return CRGPU_OK;
}

/* ---- per-device context: a caching allocator ----------------------------------------------------------------------------------
 * A frame of this renderer wants ~35 GB of wavefront state, a 50 MB scene and a framebuffer.  cudaMalloc of those costs
 * 10-55 ms and cudaFree of the 35 GB 0.3-0.5 s — per FRAME when every renderFrame creates and
 * destroys its scene replica, as the reference's renderFrame does with its buffers.  So device memory released by a scene goes
 * back to a per-device cache and the next scene on that device takes it from there (best fit within 2x); a cudaMalloc that
 * fails trims the cache and retries.  crgpu_device_trim() hands everything back to the driver. */
#define CRG_MAX_DEVICES 64
struct Cached { void *p; size_t bytes; };
struct DevCtx {
	std::mutex lock;
	std::vector<Cached> cache;
	size_t cached = 0;
};
static DevCtx g_ctx[CRG_MAX_DEVICES];
static DevCtx &ctx_of(int dev) { return g_ctx[dev >= 0 && dev < CRG_MAX_DEVICES ? dev : 0]; }

static void ctx_trim_locked(DevCtx &c) {
	for (Cached &b : c.cache) cudaFree(b.p);
	c.cache.clear();
	c.cached = 0;
}
/* the calling thread's current device must be `dev` */
static int ctx_alloc(int dev, size_t bytes, void **out) {
	*out = nullptr;
	if (bytes == 0) bytes = 256;
	DevCtx &c = ctx_of(dev);
	std::lock_guard<std::mutex> g(c.lock);
	int best = -1;
	for (size_t i = 0; i < c.cache.size(); ++i)
		if (c.cache[i].bytes >= bytes && c.cache[i].bytes <= 2 * bytes + (1u << 20) && (best < 0 || c.cache[i].bytes < c.cache[(size_t)best].bytes)) best = (int)i;
	if (best >= 0) {
		*out = c.cache[(size_t)best].p;
		c.cached -= c.cache[(size_t)best].bytes;
		c.cache.erase(c.cache.begin() + best);
		return CRGPU_OK;
	}
	cudaError_t e = cudaMalloc(out, bytes);
	if (e == cudaErrorMemoryAllocation && !c.cache.empty()) {
		cudaGetLastError();
		ctx_trim_locked(c);
		e = cudaMalloc(out, bytes);
	}
	if (e == cudaErrorMemoryAllocation) { cudaGetLastError(); *out = nullptr; return fail(CRGPU_ERR_NOMEM, "out of device memory allocating %zu bytes on device %d", bytes, dev); }
	if (e != cudaSuccess) { *out = nullptr; return fail(CRGPU_ERR_CUDA, "cudaMalloc(%zu): %s", bytes, cudaGetErrorString(e)); }
	return CRGPU_OK;
}
/* size actually backing a pointer handed out for a request of `bytes` is not tracked: callers remember their request, and a
 * cached block is re-used only for requests it can hold, so recording the REQUEST size is conservative and safe */
static void ctx_free(int dev, void *p, size_t bytes) {
	if (!p) return;
	if (bytes == 0) bytes = 256;
	DevCtx &c = ctx_of(dev);
	std::lock_guard<std::mutex> g(c.lock);
	if (c.cache.size() >= 24) {                      /* bound the list: drop the smallest entry */
		size_t k = 0;
		for (size_t i = 1; i < c.cache.size(); ++i) if (c.cache[i].bytes < c.cache[k].bytes) k = i;
		cudaFree(c.cache[k].p);
		c.cached -= c.cache[k].bytes;
		c.cache.erase(c.cache.begin() + (long)k);
	}
	c.cache.push_back({ p, bytes });
	c.cached += bytes;
}
static size_t ctx_cached_bytes(int dev) { DevCtx &c = ctx_of(dev); std::lock_guard<std::mutex> g(c.lock); return c.cached; }

/* One allocation from the per-device cache, which it goes back to when the owner is destroyed, overwritten or released. */
struct DevBlock {
	int dev = 0;
	void *p = nullptr;
	size_t bytes = 0;
	DevBlock() = default;
	DevBlock(DevBlock &&o) noexcept : dev(o.dev), p(o.p), bytes(o.bytes) { o.p = nullptr; o.bytes = 0; }
	DevBlock &operator=(DevBlock &&o) noexcept {
		if (this != &o) { release(); dev = o.dev; p = o.p; bytes = o.bytes; o.p = nullptr; o.bytes = 0; }
		return *this;
	}
	~DevBlock() { release(); }
	void release() { ctx_free(dev, p, bytes); p = nullptr; bytes = 0; }
	/* releases the block it holds, then takes one of `n` bytes on `device` (the calling thread's current device); empty on failure */
	int alloc(int device, size_t n) {
		release();
		dev = device;
		int rc = ctx_alloc(device, n, &p);
		if (!rc) bytes = n;
		return rc;
	}
	template <class T> T *as() const { return static_cast<T *>(p); }
};

extern "C" int crgpu_device_trim(int device) {
	int ndev = 0;
	int rc = crgpu_device_count(&ndev);
	if (rc) return rc;
	if (device < 0 || device >= ndev) return fail(CRGPU_ERR_BAD_ARGUMENT, "device %d out of range (have %d)", device, ndev);
	CU(cudaSetDevice(device));
	DevCtx &c = ctx_of(device);
	std::lock_guard<std::mutex> g(c.lock);
	ctx_trim_locked(c);
	return CRGPU_OK;
}

/* pinned host memory for buffers that cross PCIe every frame (the host framebuffer of renderFrame, the prepared scene) */
extern "C" void *crgpu_host_alloc(size_t bytes) {
	void *p = nullptr;
	if (cudaHostAlloc(&p, bytes ? bytes : 1, cudaHostAllocPortable) != cudaSuccess) { cudaGetLastError(); return nullptr; }
	return p;
}
extern "C" void crgpu_host_free(void *p) { if (p) cudaFreeHost(p); }

/* ---- the prepared scene: the flat scene re-laid out for the kernels, in ONE host slab (pinned) ----------------------------------
 * crgpu_prepare() does everything about a scene that does not depend on the device: validation, BVH re-layout into pair nodes,
 * triangle packing, shading records.  crgpu_scene_create_prepared() is then one host->device copy of the slab plus two small
 * pointer-carrying tables.  A host that renders many frames of one scene, or one frame on many GPUs, prepares once. */
enum { SEC_STAGE, SEC_PAIRS, SEC_TRIS, SEC_SLOT_POLY, SEC_KEYS, SEC_SPOLYS, SEC_TOP_ITEMS, SEC_BVHS, SEC_INSTS, SEC_MATS, SEC_FLAT, SEC_ORDER, SEC_NODES, SEC_TEXS, SEC_LUT,
       SEC_TEXDATA, SEC_COUNT };
/* What the geometry edits (crgpu_scene_set_instances, crgpu_scene_set_meshes, crgpu_scene_set_instance_list) need beyond the slab:
 * the records they check an edit against, the BVH root bounds they build the top level from, and the objects a new instance list
 * may instance. */
struct EditRecord {
	std::vector<uint32_t> inst_kind, inst_object;   /* kind and object of every instance of the current list */
	std::vector<uint32_t> last;                      /* the last instance of each instance's object: all of them take its ray offset */
	std::vector<float> bvh_root;                     /* root bounds of every BVH as stored, 6 floats each (the slab keeps only pair
	                                                    nodes, whose roots' own boxes are not in it); an edited scene keeps them current */
	std::vector<crs_mesh> meshes;                    /* every mesh record: an edit must keep each */
	std::vector<crs_sphere> spheres;                 /* every sphere record: radius and material of its instances */
	std::vector<uint32_t> bvh_prims;                 /* primitives of each BVH */
};
struct crgpu_prepared {
	crs_prefs prefs;
	crs_camera camera;
	int32_t background;
	uint32_t instance_count;
	DevBvh top;
	float world_lo[3], world_inv[3];
	uint32_t stage_pairs;
	uint32_t texture_count;
	size_t key_inst_off;       /* the instance keys follow the prim-slot keys in SEC_KEYS */
	uint32_t material_count;
	uint32_t flat_keys;        /* DevScene::flat_keys */
	bool xnodes;               /* some node is of a kind only the complete interpreter (NodeX) evaluates */
	DevFlatBg bg;              /* DevScene::bg */
	uint8_t *slab;
	bool pinned;
	size_t slab_bytes;
	size_t off[SEC_COUNT], len[SEC_COUNT];
	EditRecord rec;
};

/* The parts of an edited scene's instance block: the last-instance table and the top level's item records, then, from the first
 * instance-list edit on, the scene's own instance records and instance keys (DevScene::instances and inst_key point at them in place
 * of the slab's SEC_INSTS and key tail). */
struct InstParts {
	uint32_t *last;
	DevTopItem *items;
	DevInstance *recs;         /* NULL before the first list edit */
	uint8_t *keys;             /* NULL before the first list edit */
};

struct crgpu_scene {
	int device = 0;
	int sm_count = 0;
	bool xnodes = false;       /* crgpu_prepared::xnodes: selects the K3 / tail kernels with the complete node interpreter */
	cudaStream_t stream = nullptr;   /* the stream work is enqueued on (own_stream unless crgpu_set_stream) */
	cudaStream_t own_stream = nullptr;
	unsigned long long fetched[8] = {};   /* device counters at the previous stats fetch */
	uint64_t pend_paths = 0, pend_launches = 0;
	float pend_trace_ms = 0.f, pend_shade_ms = 0.f, pend_total_ms = 0.f;
	DevScene dev = {};
	DevScene *dev_copy = nullptr;    /* the same descriptor in HBM, for kernels that call noinline device functions */
	DevBlock slab;                   /* the scene arrays + dev_copy */
	DevBlock small;                  /* hist, counts, stats */
	DevBlock fb;                     /* W*H*3 fp32, row H-1-y */
	DevBlock fb8;                    /* sRGB8 staging, allocated when first used (alloc_srgb8) */
	size_t fb_floats = 0;
	uint64_t max_paths = 0;
	uint64_t cap_paths = 0;          /* capacity of the wavefront buffers */
	DevBlock wave;
	int wave_sets = 0;               /* 1, or 2 when batches are overlapped on two streams (each set holds cap_paths paths) */
	WaveBuffers wb = {};             /* set 0 */
	WaveBuffers wb2 = {};            /* set 1: own ray / hit / radiance buffers and own hist + counts; stats shared */
	cudaStream_t stream2 = nullptr;  /* the second stream of overlapped batches */
	cudaEvent_t ev[4] = {};
	cudaEvent_t evAcc[2] = {}, evFork = nullptr;   /* accumulate-order chain between the two streams */
	DevBlock pixels;                 /* device pixel list of the last crgpu_render_tiles tile set */
	std::vector<int> pixel_key;
	bool armed = false;              /* crgpu_stop_enable: render calls run the stop gates and the ordered commit */
	unsigned *stop_host = nullptr;   /* pinned, mapped: [0] stop request, [1] committed pass index, [2] a call is in flight, [3] snapshot
	                                    state (0 idle, 1 requested, 2 staged), [4] its pass index (NULL until armed once) */
	unsigned *stop_ctl = nullptr;    /* device: [0] pass index the running average has reached, [1], [2] abandoned flags of the wave sets,
	                                    [3] the next publish step stages a snapshot, [4] its block count (crgpu_wave.cuh) */
	DevBlock snap8;                  /* W*H*3 sRGB8 snapshot staged by a publish step (allocated by the first armed call) */
	cudaStream_t snap_stream = nullptr;   /* crgpu_take_snapshot's copies: never behind the render (created when first armed) */
	/* scene edits */
	EditRecord rec;                  /* crgpu_prepared::rec */
	std::vector<DevBvh> bvhs;        /* the committed BVH records (the slab's copy is what the kernels read) */
	std::vector<uint32_t> stage_cap; /* staged pairs reserved for each BVH at upload */
	std::vector<uint32_t> mesh_region;   /* first pair of a mesh's own region in the pairs block (UINT32_MAX: none yet) */
	uint32_t pair_count = 0;         /* pair nodes uploaded */
	uint32_t pair_cap = 0;           /* pair nodes dev.pairs holds: pair_count until the first geometry edit, then the pairs block's */
	uint32_t top_off = 0, top_cap = 0;   /* the top region in the pairs block: first pair and room, at least max(1, n - 1) for the current
	                                        n instances (reserved behind the uploaded pairs until a list outgrows it) */
	uint32_t top_stage_cap = 0;      /* staged top-level pairs reserved at upload */
	uint32_t material_count = 0;     /* as uploaded or as the last crgpu_scene_add_objects left it: a shading edit must keep it */
	uint32_t mat_cap = 0;            /* materials dev.materials and dev.flat have room for */
	uint32_t slot_count = 0, poly_count = 0;             /* triangle slots and polys of the scene */
	uint32_t slot_cap = 0, poly_cap = 0, bvh_cap = 0;    /* room of the geometry sections dev points at (GeomParts) */
	DevBlock geom;                   /* NULL until the first add: the geometry block (GeomParts), in place of the slab's sections */
	DevBlock mats;                   /* NULL until an add outgrows the uploaded materials: the materials block (MatParts) */
	DevBlock pairs;                  /* NULL until the first geometry edit: the uploaded pairs, the top region, the edited meshes' regions */
	DevBlock insts;                  /* NULL until the first geometry edit: the instance block (InstParts) */
	InstParts ip = {};               /* its parts */
	uint32_t inst_cap = 0;           /* instances it has room for */
	DevBlock scratch;                /* a geometry edit's inputs, records and builder scratch; grows only, and nothing in it outlives a call */
	DevBlock shade;                  /* NULL until the first shading edit: the node graph, texture table and texel data the kernels read in
	                                    place of the slab's */
	/* views (crgpu_scene_set_views): view 0 is the scene's camera and framebuffer; views 1 .. view_count - 1 live in the views block */
	uint32_t view_count = 1;
	uint32_t view_cap = 1;           /* views the block has room for (1: no block) */
	DevBlock views;                  /* NULL until the first set_views of more than one view: view_cap - 1 cameras, then view_cap - 1
	                                    framebuffers (views_layout); grows only */
	/* adaptive rounds (crgpu_adaptive_reset / _round / _read) */
	DevBlock adapt;                  /* NULL until the first reset and after a size change: view 0's pixel records, the active list and
	                                    the select's scan scratch (AdaptParts) */
	unsigned *adapt_host = nullptr;  /* pinned, mapped: [0] active count, [1] min and [2] max count of the last select */
	std::vector<int> adapt_key;      /* the last tile set found to have no overlapping tiles */
};

/* K1 and K2 take the host descriptor s->dev by value; K3, the tail kernel and the KAT read its HBM copy s->dev_copy.  Writes the
 * copy and waits for it (and for everything queued before it on the scene's stream). */
static int publish(crgpu_scene *s) {
	CU(cudaMemcpyAsync(s->dev_copy, &s->dev, sizeof(DevScene), cudaMemcpyHostToDevice, s->stream));
	CU(cudaStreamSynchronize(s->stream));
	return CRGPU_OK;
}

/* fb8 or snap8, an sRGB8 staging buffer of the image, when first used */
static int alloc_srgb8(crgpu_scene *s, DevBlock &b) { return b.p ? CRGPU_OK : b.alloc(s->device, s->fb_floats); }

/* ---- node graph checks -------------------------------------------------------------------------------------- */
static bool node_ok(const crs_scene *f, int idx) { return idx >= 0 && (uint32_t)idx < f->node_count; }

/* Nesting as the device counts it (crgpu_shade.cuh).  The hot interpreter NodeEval<CRG_NODE_DEPTH> knows the node kinds of JSON
 * scenes: color->value->color recursion costs a level at checker/blackbody -> value (grayscale/alpha -> color and the checker's
 * A/B tail calls are free).  At the first node of any other kind the complete interpreter NodeX<CRG_XNODE_DEPTH> takes over, where
 * EVERY edge costs a level (xnode_depth) whatever the kinds below. */
static int xnode_depth(const crs_scene *f, int idx, int guard) {
	if (!node_ok(f, idx) || guard > 64) return 1000;
	const crs_node &n = f->nodes[idx];
	int ins = 0;
	switch (n.kind) {
	case CRS_COLOR_CONSTANT: case CRS_COLOR_IMAGE: case CRS_COLOR_GRADIENT: case CRS_VALUE_CONSTANT: case CRS_VALUE_RAYLENGTH:
	case CRS_VECTOR_CONSTANT: case CRS_VECTOR_NORMAL: return 0;
	case CRS_COLOR_CHECKER: case CRS_COLOR_COMBINE_RGB: ins = 3; break;
	case CRS_VALUE_MATH: if (n.options >= CRS_MATH_OP_COUNT) return 1000; ins = 2; break;
	case CRS_VECTOR_VECMATH: if (n.options >= CRS_VEC_OP_COUNT) return 1000; ins = 2; break;
	case CRS_COLOR_BLACKBODY: case CRS_COLOR_COMBINE_VALUE: case CRS_COLOR_VECTOCOLOR: case CRS_VALUE_GRAYSCALE: case CRS_VALUE_ALPHA: ins = 1; break;
	case CRS_VALUE_FRESNEL: {                            /* in1 (normal) is never evaluated (fresnel.c:43-55) but must be a vector node */
		if (!node_ok(f, n.in[1])) return 1000;
		const int k = f->nodes[n.in[1]].kind;
		if (k != CRS_VECTOR_CONSTANT && k != CRS_VECTOR_NORMAL && k != CRS_VECTOR_VECMATH) return 1000;
		ins = 1; break;
	}
	default: return 1000;
	}
	/* operand classes: what each input must be */
	int m = 0;
	for (int k = 0; k < ins; ++k) {
		if (!node_ok(f, n.in[k])) return 1000;
		const int ck = f->nodes[n.in[k]].kind;
		const bool is_color = ck >= CRS_COLOR_CONSTANT && ck <= CRS_COLOR_COMBINE_RGB, is_value = ck >= CRS_VALUE_CONSTANT && ck <= CRS_VALUE_RAYLENGTH,
				   is_vector = ck >= CRS_VECTOR_CONSTANT && ck <= CRS_VECTOR_VECMATH;
		bool ok;
		switch (n.kind) {
		case CRS_COLOR_CHECKER: ok = k < 2 ? is_color : is_value; break;
		case CRS_VALUE_GRAYSCALE: case CRS_VALUE_ALPHA: ok = is_color; break;
		case CRS_COLOR_VECTOCOLOR: case CRS_VECTOR_VECMATH: ok = is_vector; break;
		default: ok = is_value; break;                   /* blackbody, combine, combine rgb, math, fresnel (IOR) */
		}
		if (!ok) return 1000;
		const int d = xnode_depth(f, n.in[k], guard + 1);
		if (d > m) m = d;
	}
	return 1 + m;
}
static int xnode_entry(const crs_scene *f, int idx, int guard) { return xnode_depth(f, idx, guard) <= CRG_XNODE_DEPTH ? 0 : 1000; }
static int value_depth(const crs_scene *f, int idx, int guard);
static int color_depth(const crs_scene *f, int idx, int guard) {
	if (!node_ok(f, idx) || guard > 64) return 1000;
	const crs_node &n = f->nodes[idx];
	switch (n.kind) {
	case CRS_COLOR_CONSTANT: case CRS_COLOR_IMAGE: case CRS_COLOR_GRADIENT: return 0;
	case CRS_COLOR_CHECKER: {
		int a = color_depth(f, n.in[0], guard + 1), b = color_depth(f, n.in[1], guard + 1);
		int v = 1 + value_depth(f, n.in[2], guard + 1);
		int m = a > b ? a : b;
		return m > v ? m : v;
	}
	case CRS_COLOR_BLACKBODY: return 1 + value_depth(f, n.in[0], guard + 1);
	case CRS_COLOR_VECTOCOLOR: case CRS_COLOR_COMBINE_VALUE: case CRS_COLOR_COMBINE_RGB: return xnode_entry(f, idx, guard);
	default: return 1000;
	}
}
static int value_depth(const crs_scene *f, int idx, int guard) {
	if (!node_ok(f, idx) || guard > 64) return 1000;
	const crs_node &n = f->nodes[idx];
	switch (n.kind) {
	case CRS_VALUE_CONSTANT: return 0;
	case CRS_VALUE_GRAYSCALE: case CRS_VALUE_ALPHA: return color_depth(f, n.in[0], guard + 1);
	case CRS_VALUE_MATH: case CRS_VALUE_FRESNEL: case CRS_VALUE_RAYLENGTH: return xnode_entry(f, idx, guard);
	default: return 1000;
	}
}
static bool color_reads_uv(const crs_scene *f, int idx);
static bool value_reads_uv(const crs_scene *f, int idx) {
	if (!node_ok(f, idx)) return false;
	const crs_node &n = f->nodes[idx];
	switch (n.kind) {
	case CRS_VALUE_GRAYSCALE: case CRS_VALUE_ALPHA: return color_reads_uv(f, n.in[0]);
	case CRS_VALUE_MATH: return value_reads_uv(f, n.in[0]) || value_reads_uv(f, n.in[1]);
	case CRS_VALUE_FRESNEL: return value_reads_uv(f, n.in[0]);
	default: return false;
	}
}
static bool color_reads_uv(const crs_scene *f, int idx) {
	if (!node_ok(f, idx)) return false;
	const crs_node &n = f->nodes[idx];
	switch (n.kind) {
	case CRS_COLOR_IMAGE: case CRS_COLOR_CHECKER: return true;
	case CRS_COLOR_BLACKBODY: case CRS_COLOR_COMBINE_VALUE: return value_reads_uv(f, n.in[0]);
	case CRS_COLOR_COMBINE_RGB: return value_reads_uv(f, n.in[0]) || value_reads_uv(f, n.in[1]) || value_reads_uv(f, n.in[2]);
	default: return false;            /* vector nodes never read uv */
	}
}
/* validates a bsdf tree; *add_depth = nesting of ADD nodes; *uv = some node reads uv */
static int check_bsdf(const crs_scene *f, int idx, int add_level, int guard, bool *uv) {
	if (!node_ok(f, idx) || guard > 64) return fail(CRGPU_ERR_UNSUPPORTED, "bsdf node index %d out of range or graph too deep", idx);
	const crs_node &n = f->nodes[idx];
	auto col = [&](int c) -> int {
		if (color_depth(f, c, 0) > CRG_NODE_DEPTH) return fail(CRGPU_ERR_UNSUPPORTED, "color node %d nests deeper than %d", c, CRG_NODE_DEPTH);
		if (color_reads_uv(f, c)) *uv = true;
		return 0;
	};
	auto val = [&](int v) -> int {
		if (value_depth(f, v, 0) > CRG_NODE_DEPTH) return fail(CRGPU_ERR_UNSUPPORTED, "value node %d nests deeper than %d", v, CRG_NODE_DEPTH);
		if (value_reads_uv(f, v)) *uv = true;
		return 0;
	};
	int rc;
	switch (n.kind) {
	case CRS_BSDF_DIFFUSE: case CRS_BSDF_TRANSPARENT: case CRS_BSDF_ISOTROPIC: return col(n.in[0]);
	case CRS_BSDF_METAL: case CRS_BSDF_EMISSIVE: if ((rc = col(n.in[0]))) return rc; return val(n.in[1]);
	case CRS_BSDF_GLASS: case CRS_BSDF_BACKGROUND:
		if ((rc = col(n.in[0]))) return rc; if ((rc = val(n.in[1]))) return rc; return val(n.in[2]);
	case CRS_BSDF_PLASTIC:
		if ((rc = col(n.in[0]))) return rc; if ((rc = col(n.in[1]))) return rc;
		return check_bsdf(f, n.in[2], add_level, guard + 1, uv);
	case CRS_BSDF_MIX:
		if ((rc = val(n.in[2]))) return rc;
		if ((rc = check_bsdf(f, n.in[0], add_level, guard + 1, uv))) return rc;
		return check_bsdf(f, n.in[1], add_level, guard + 1, uv);
	case CRS_BSDF_ADD:
		if (2 * (add_level + 1) > CRG_ADD_STACK) return fail(CRGPU_ERR_UNSUPPORTED, "ADD nodes nest deeper than %d", CRG_ADD_STACK / 2);
		if ((rc = check_bsdf(f, n.in[0], add_level + 1, guard + 1, uv))) return rc;
		return check_bsdf(f, n.in[1], add_level + 1, guard + 1, uv);
	default: return fail(CRGPU_ERR_UNSUPPORTED, "node %d has kind %d where a bsdf is expected", idx, n.kind);
	}
}

/* ---- flat materials (DevFlat): the fixed-form graphs the flat K3 launch samples without the node interpreter -------------
 * A leaf (diffuse, metal, glass, emissive, or plastic over a diffuse) whose colour is a constant or one image node and whose values
 * are constants, alone or under the loader's legacy wrapper Mix(Transparent(constant c0), leaf, Alpha(constant or image colour))
 * (host/loader/cr_nodes.c crl_assign_bsdf).  Folding copies the bits the interpreter would read — f[0..3] of a constant colour, f[0]
 * of a value, f[3] of an alpha's constant, tex / options of an image — and computes nothing.  Anything else stays generic. */
static bool flat_color(const crs_scene *f, int idx, float col[4], int32_t &tex, uint32_t &opt, bool &img) {
	if (!node_ok(f, idx)) return false;
	const crs_node &n = f->nodes[idx];
	if (n.kind == CRS_COLOR_CONSTANT) { memcpy(col, n.f, 4 * sizeof(float)); img = false; return true; }
	if (n.kind == CRS_COLOR_IMAGE) { tex = n.tex; opt = n.options; img = true; return true; }
	return false;
}
static bool flat_value(const crs_scene *f, int idx, float &v) {
	if (!node_ok(f, idx) || f->nodes[idx].kind != CRS_VALUE_CONSTANT) return false;
	memcpy(&v, &f->nodes[idx].f[0], sizeof v);
	return true;
}
static bool flat_leaf(const crs_scene *f, int idx, DevFlat &d) {
	if (!node_ok(f, idx)) return false;
	const crs_node &n = f->nodes[idx];
	int color = n.in[0];
	switch (n.kind) {
	case CRS_BSDF_DIFFUSE: d.kind = CRG_FLAT_DIFFUSE; break;
	case CRS_BSDF_METAL: d.kind = CRG_FLAT_METAL; if (!flat_value(f, n.in[1], d.rough)) return false; break;
	case CRS_BSDF_GLASS:
		d.kind = CRG_FLAT_GLASS;
		if (!flat_value(f, n.in[1], d.rough) || !flat_value(f, n.in[2], d.ior)) return false;
		break;
	case CRS_BSDF_EMISSIVE: d.kind = CRG_FLAT_EMISSIVE; if (!flat_value(f, n.in[1], d.strength)) return false; break;
	case CRS_BSDF_PLASTIC: {                          /* roughness = color(in[1]).r; in[0] is never read (plastic.c:42-87) */
		d.kind = CRG_FLAT_PLASTIC;
		if (!node_ok(f, n.in[1]) || f->nodes[n.in[1]].kind != CRS_COLOR_CONSTANT) return false;
		memcpy(&d.rough, &f->nodes[n.in[1]].f[0], sizeof d.rough);
		if (!node_ok(f, n.in[2]) || f->nodes[n.in[2]].kind != CRS_BSDF_DIFFUSE) return false;
		color = f->nodes[n.in[2]].in[0];
		break;
	}
	default: return false;
	}
	bool img = false;
	if (!flat_color(f, color, d.col, d.col_tex, d.col_opt, img)) return false;
	if (img) d.flags |= CRG_FLAT_COL_IMG;
	return true;
}
static DevFlat fold_flat(const crs_scene *f, int root) {
	DevFlat d;
	memset(&d, 0, sizeof d);
	int leaf = root;
	const crs_node &r = f->nodes[root];
	if (r.kind == CRS_BSDF_MIX) {                     /* only the wrapper's shape: MIX(TRANSPARENT(constant), leaf, ALPHA(colour)) */
		bool ok = node_ok(f, r.in[0]) && node_ok(f, r.in[2]);
		if (ok) {
			const crs_node &t = f->nodes[r.in[0]], &a = f->nodes[r.in[2]];
			ok = t.kind == CRS_BSDF_TRANSPARENT && node_ok(f, t.in[0]) && f->nodes[t.in[0]].kind == CRS_COLOR_CONSTANT && a.kind == CRS_VALUE_ALPHA;
			float ac[4];
			bool img = false;
			if (ok) ok = flat_color(f, a.in[0], ac, d.alpha_tex, d.alpha_opt, img);
			if (ok) {
				memcpy(d.c0, f->nodes[t.in[0]].f, sizeof d.c0);
				if (img) d.flags |= CRG_FLAT_ALPHA_IMG;
				else memcpy(&d.alpha, &ac[3], sizeof d.alpha);
				d.flags |= CRG_FLAT_WRAPPED;
			}
		}
		if (!ok) { memset(&d, 0, sizeof d); return d; }
		leaf = r.in[1];
	}
	if (!flat_leaf(f, leaf, d)) memset(&d, 0, sizeof d);
	return d;
}

/* ---- the folded background (DevFlatBg): BACKGROUND(constant | image | gradient colour, constant strength, constant offset) ---------
 * host/loader/cr_sceneload.c builds every JSON scene's background in this form (crl_background).  Folding copies the node fields
 * cr_sample_background reads and computes nothing; any other graph stays with the interpreter (kind CRG_BG_NONE). */
static DevFlatBg fold_background(const crs_scene *f, int root) {
	DevFlatBg b;
	memset(&b, 0, sizeof b);
	const crs_node &r = f->nodes[root];
	if (!flat_value(f, r.in[1], b.strength) || !flat_value(f, r.in[2], b.offset) || !node_ok(f, r.in[0])) { memset(&b, 0, sizeof b); return b; }
	const crs_node &c = f->nodes[r.in[0]];
	switch (c.kind) {
	case CRS_COLOR_CONSTANT: b.kind = CRG_BG_CONSTANT; break;
	case CRS_COLOR_IMAGE: b.kind = CRG_BG_IMAGE; b.tex = c.tex; b.opt = c.options; break;
	case CRS_COLOR_GRADIENT: b.kind = CRG_BG_GRADIENT; break;
	default: memset(&b, 0, sizeof b); return b;
	}
	memcpy(b.f, c.f, sizeof b.f);
	return b;
}

/* ---- the shading fold: everything the kernels read about materials, the node graph, textures and the background --------------
 * crgpu_prepare and crgpu_scene_set_shading both take these records from here, so an edited scene holds the bytes a fresh prepare
 * of the same arrays would.  Reads material_count, materials, node_count, nodes, texture_count, textures, texdata_bytes and
 * background of `f`; validates them as an upload must (the error is the one crgpu_prepare returns). */
struct ShadingFold {
	bool xnodes;                       /* some node is of a kind only the complete interpreter (NodeX) evaluates */
	DevFlatBg bg;
	std::vector<DevMaterial> mats;
	std::vector<DevFlat> flat;
	std::vector<DevTexture> texs;      /* data = byte offset into texdata (patched with a device address at upload) */
	std::vector<uint8_t> order;        /* K4's bucket order, 256 keys */
	uint32_t flat_keys;
};

static int fold_shading(const crs_scene *f, ShadingFold &out) {
	if (!node_ok(f, f->background) || f->nodes[f->background].kind != CRS_BSDF_BACKGROUND)
		return fail(CRGPU_ERR_UNSUPPORTED, "scene background must be a background node");
	out.xnodes = false;
	for (uint32_t i = 0; i < f->node_count; ++i) {
		const int k = f->nodes[i].kind;
		if (k == CRS_COLOR_VECTOCOLOR || k == CRS_COLOR_COMBINE_VALUE || k == CRS_COLOR_COMBINE_RGB || k == CRS_VALUE_MATH || k == CRS_VALUE_FRESNEL ||
			k == CRS_VALUE_RAYLENGTH || k == CRS_VECTOR_CONSTANT || k == CRS_VECTOR_NORMAL || k == CRS_VECTOR_VECMATH) out.xnodes = true;
	}
	out.bg = fold_background(f, f->background);
	int rc;
	{
		bool uv = false;
		if ((rc = check_bsdf(f, f->background, 0, 0, &uv))) return rc;
	}
	out.mats.resize(f->material_count);
	out.flat.resize(f->material_count);
	for (uint32_t i = 0; i < f->material_count; ++i) {
		const crs_material &m = f->materials[i];
		bool uv = false;
		if ((rc = check_bsdf(f, m.bsdf, 0, 0, &uv))) return rc;
		DevMaterial d;
		memset(&d, 0, sizeof d);
		d.emission[0] = m.emission[0]; d.emission[1] = m.emission[1]; d.emission[2] = m.emission[2];
		d.IOR = m.IOR; d.bsdf = m.bsdf;
		/* x + w*0 == x bit-for-bit for finite w, so only non-zero (or non-finite) emission needs the add */
		const bool emits = !(m.emission[0] == 0.0f && m.emission[1] == 0.0f && m.emission[2] == 0.0f);
		d.flags = (uv ? 1u : 0u) | (emits ? 2u : 0u);
		out.mats[i] = d;
		out.flat[i] = fold_flat(f, m.bsdf);
	}
	out.texs.resize(f->texture_count);
	for (uint32_t i = 0; i < f->texture_count; ++i) {
		const crs_texture &t = f->textures[i];
		const uint64_t bytes = (uint64_t)t.width * t.height * t.channels * (t.is_float ? 4u : 1u);
		if (t.width == 0 || t.height == 0 || t.channels == 0 || t.channels > 4 || t.width > 65536u || t.height > 65536u ||
			t.data_offset > f->texdata_bytes || bytes > f->texdata_bytes - t.data_offset) {
			return fail(CRGPU_ERR_BAD_ARGUMENT, "texture %u malformed", i);
		}
		DevTexture d;
		d.width = t.width; d.height = t.height; d.channels = t.channels; d.is_float = t.is_float; d.has_alpha = t.has_alpha; d.pad = 0;
		d.wmask = (t.width & (t.width - 1u)) == 0u ? t.width - 1u : 0u;
		d.hmask = (t.height & (t.height - 1u)) == 0u ? t.height - 1u : 0u;
		d.data = reinterpret_cast<const uint8_t *>((uintptr_t)t.data_offset);
		out.texs[i] = d;
	}
	for (uint32_t i = 0; i < f->node_count; ++i)
		if (f->nodes[i].kind == CRS_COLOR_IMAGE && (f->nodes[i].tex >= (int32_t)f->texture_count || f->nodes[i].tex < -1))
			return fail(CRGPU_ERR_BAD_ARGUMENT, "node %u texture index out of range", i);
	/* K4's bucket order for the flat launch: the misses, the keys of flat materials (1..254, one material each), then the rest —
	 * the generic keys and the overflow key 255, which materials 254 and up share */
	auto is_flat = [&](uint32_t k) { return k < 255u && k - 1u < f->material_count && out.flat[k - 1u].kind != CRG_FLAT_NONE; };
	out.order.clear();
	out.order.push_back(0);
	for (uint32_t k = 1; k < 256; ++k) if (is_flat(k)) out.order.push_back((uint8_t)k);
	out.flat_keys = (uint32_t)out.order.size() - 1u;
	for (uint32_t k = 1; k < 256; ++k) if (!is_flat(k)) out.order.push_back((uint8_t)k);
	return CRGPU_OK;
}

/* ---- BVH re-layout: reference nodes (bvh.c:37-42) -> BFS-ordered PairNodes ---------------------------------------- */
/* errors raised on worker threads (fail() writes a thread-local buffer): first one wins, reported by the caller */
struct HostError {
	std::mutex lock;
	int code = 0;
	char msg[256] = "";
	int set(int c, const char *m) { std::lock_guard<std::mutex> g(lock); if (!code) { code = c; snprintf(msg, sizeof msg, "%s", m); } return c; }
};

/* fn(lo, hi) over [0, n) on a few host threads (CRGPU_HOST_THREADS, default min(hardware, 16)); small n stays inline */
template <class F>
static void host_parallel_for(uint32_t n, F fn) {
	static const unsigned want = [] {
		const char *e = getenv("CRGPU_HOST_THREADS");
		unsigned t = e ? (unsigned)atoi(e) : std::thread::hardware_concurrency();
		return t < 1u ? 1u : (t > 16u ? 16u : t);
	}();
	const unsigned threads = n < 16384u ? 1u : want;
	if (threads <= 1u) { fn(0u, n); return; }
	std::vector<std::thread> pool;
	for (unsigned k = 1; k < threads; ++k)
		pool.emplace_back(fn, (uint32_t)((uint64_t)n * k / threads), (uint32_t)((uint64_t)n * (k + 1) / threads));
	fn(0u, (uint32_t)((uint64_t)n / threads));
	for (auto &t : pool) t.join();
}

/* ---- instance packing: the DevInstance records, the sphere instances' shading keys and the last-instance table of a list ----------
 * crgpu_prepare and crgpu_scene_set_instance_list both take them from here.  An instance of another kind is refused with `bad_kind`
 * (crgpu_prepare: CRGPU_ERR_UNSUPPORTED, volumes; an edit: CRGPU_ERR_BAD_ARGUMENT), an object or a sphere material out of range with
 * CRGPU_ERR_BAD_ARGUMENT.  ray_offset is the object's as loaded; the top-level build on the device recomputes it. */
struct InstancePack {
	std::vector<DevInstance> recs;
	std::vector<uint8_t> keys;         /* min(material + 1, 255) of a sphere instance, 0 for a mesh instance */
	std::vector<uint32_t> last;
};
static uint8_t shade_key(uint32_t material) { return (uint8_t)(material + 1u < 255u ? material + 1u : 255u); }

static int pack_instances(const crs_instance *inst, uint32_t n, const crs_sphere *spheres, uint32_t sphere_count, const crs_mesh *meshes,
                          uint32_t mesh_count, uint32_t material_count, int bad_kind, InstancePack &out) {
	std::vector<uint32_t> last_of[2] = { std::vector<uint32_t>(mesh_count), std::vector<uint32_t>(sphere_count) };   /* by kind, object */
	for (uint32_t i = 0; i < n; ++i) {
		const crs_instance &src = inst[i];
		if (src.kind == CRS_INST_MESH) {
			if (src.object >= mesh_count) return fail(CRGPU_ERR_BAD_ARGUMENT, "instance mesh index out of range");
		} else if (src.kind == CRS_INST_SPHERE) {
			if (src.object >= sphere_count) return fail(CRGPU_ERR_BAD_ARGUMENT, "instance sphere index out of range");
			if (spheres[src.object].material >= material_count) return fail(CRGPU_ERR_BAD_ARGUMENT, "sphere material out of range");
		} else {
			return fail(bad_kind, "instance %u has kind %u (volumes are not reachable from the scene loader)", i, src.kind);
		}
		last_of[src.kind == CRS_INST_SPHERE][src.object] = i;
	}
	out.recs.resize(n);
	out.keys.assign(n, 0u);
	out.last.resize(n);
	host_parallel_for(n, [&](uint32_t lo, uint32_t hi) {
		for (uint32_t i = lo; i < hi; ++i) {
			const crs_instance &src = inst[i];
			DevInstance d;
			memset(&d, 0, sizeof d);
			memcpy(d.Ainv, src.Ainv, sizeof d.Ainv);
			memcpy(d.A, src.A, sizeof d.A);
			d.kind = src.kind;
			if (src.kind == CRS_INST_MESH) {
				d.bvh = meshes[src.object].bvh;
				d.ray_offset = meshes[src.object].ray_offset;
			} else {
				d.ray_offset = spheres[src.object].ray_offset;
				d.radius = spheres[src.object].radius;
				d.material = spheres[src.object].material;
				out.keys[i] = shade_key(d.material);
			}
			out.recs[i] = d;
			out.last[i] = last_of[src.kind == CRS_INST_SPHERE][src.object];
		}
	});
	return CRGPU_OK;
}

static int build_pairs(const crs_scene *f, const crs_bvh &b, std::vector<PairNode> &pairs, DevBvh &out, uint32_t slot_offset, HostError *err) {
	memset(&out, 0, sizeof out);
	out.pair_offset = (uint32_t)pairs.size();
	out.pair_end = out.pair_offset;
	out.node_count = b.node_count;
	out.slot_offset = slot_offset;
	if (b.node_count == 0) return CRGPU_OK;
	const crs_bvh_node *nodes = f->bvh_nodes + b.node_offset;
	if (b.node_count == 1) {
		memcpy(out.root_bounds, nodes[0].bounds, sizeof out.root_bounds);
		out.root_first = nodes[0].first_child_or_prim;
		out.root_count = nodes[0].prim_count_leaf & CRS_BVH_COUNT_MASK;
		if ((uint64_t)out.root_first + out.root_count > (uint64_t)b.prim_count) return err->set(CRGPU_ERR_BAD_ARGUMENT, "BVH leaf range outside the primitive list");
		return CRGPU_OK;
	}
	/* BFS over internal nodes; pair index = BFS rank */
	std::vector<uint32_t> order;            /* reference node index of each internal node, BFS order */
	order.reserve(b.node_count / 2 + 1);
	std::vector<uint32_t> rank(b.node_count, 0xffffffffu);
	std::vector<uint8_t> depth(b.node_count, 0);   /* the traversal stack holds CRG_MAX_STACK entries per level (bvh.c:32) */
	order.push_back(0);
	rank[0] = 0;
	for (size_t head = 0; head < order.size(); ++head) {
		const crs_bvh_node &n = nodes[order[head]];
		if (n.prim_count_leaf & CRS_BVH_LEAF_BIT) return err->set(CRGPU_ERR_BAD_ARGUMENT, "BVH root/internal node is a leaf");
		const uint32_t fc = n.first_child_or_prim;
		if ((uint64_t)fc + 1u >= (uint64_t)b.node_count) return err->set(CRGPU_ERR_BAD_ARGUMENT, "BVH child index out of range");
		if (depth[order[head]] >= CRG_MAX_STACK) return err->set(CRGPU_ERR_UNSUPPORTED, "BVH deeper than 64 levels");
		for (uint32_t k = 0; k < 2; ++k) {
			const crs_bvh_node &c = nodes[fc + k];
			if (!(c.prim_count_leaf & CRS_BVH_LEAF_BIT)) {
				if (rank[fc + k] != 0xffffffffu) return err->set(CRGPU_ERR_BAD_ARGUMENT, "BVH is not a tree");
				rank[fc + k] = (uint32_t)order.size();
				depth[fc + k] = (uint8_t)(depth[order[head]] + 1);
				order.push_back(fc + k);
			} else if ((uint64_t)c.first_child_or_prim + (uint64_t)(c.prim_count_leaf & CRS_BVH_COUNT_MASK) > (uint64_t)b.prim_count) {
				return err->set(CRGPU_ERR_BAD_ARGUMENT, "BVH leaf range outside the primitive list");
			}
		}
	}
	const size_t first = pairs.size();
	pairs.resize(first + order.size());
	host_parallel_for((uint32_t)order.size(), [&](uint32_t lo, uint32_t hi) {
		for (uint32_t r = lo; r < hi; ++r) {
			const crs_bvh_node &n = nodes[order[r]];
			const uint32_t fc = n.first_child_or_prim;
			PairNode p;
			memset(&p, 0, sizeof p);
			const crs_bvh_node &l = nodes[fc], &rr = nodes[fc + 1];
			memcpy(p.lb, l.bounds, sizeof p.lb);
			memcpy(p.rb, rr.bounds, sizeof p.rb);
			if (l.prim_count_leaf & CRS_BVH_LEAF_BIT) { p.lref = l.first_child_or_prim; p.lmeta = CRG_LEAF_BIT | (l.prim_count_leaf & CRS_BVH_COUNT_MASK); }
			else { p.lref = rank[fc]; p.lmeta = 0; }
			if (rr.prim_count_leaf & CRS_BVH_LEAF_BIT) { p.rref = rr.first_child_or_prim; p.rmeta = CRG_LEAF_BIT | (rr.prim_count_leaf & CRS_BVH_COUNT_MASK); }
			else { p.rref = rank[fc + 1]; p.rmeta = 0; }
			pairs[first + r] = p;
		}
	});
	out.pair_end = (uint32_t)pairs.size();
	return CRGPU_OK;
}

static inline void f3(float *dst, const float *src, size_t idx) { dst[0] = src[3 * idx]; dst[1] = src[3 * idx + 1]; dst[2] = src[3 * idx + 2]; }

/* The world box the kernels normalise hit points by: the top-level root's bounds b (minx,maxx,miny,maxy,minz,maxz). */
static void world_box(const float b[6], float lo[3], float inv[3]) {
	for (int k = 0; k < 3; ++k) {
		const float e = b[2 * k + 1] - b[2 * k];
		lo[k] = b[2 * k];
		inv[k] = (e > 0.f && e < 3.0e38f) ? 1.0f / e : 0.f;
	}
}

static DevCamera dev_camera(const crs_camera &c) {
	DevCamera d;
	d.sensor_x = c.sensor_x; d.sensor_y = c.sensor_y; d.aperture = c.aperture; d.focal_distance = c.focal_distance;
	memcpy(d.forward, c.forward, 12); memcpy(d.right, c.right, 12); memcpy(d.up, c.up, 12);
	d.width = c.width; d.height = c.height;
	memcpy(d.A, c.A, sizeof d.A);
	return d;
}

/* all wavefront buffers of a scene are carved from ONE device block (one cudaMalloc / one cache hit per frame) */
static int alloc_wave(crgpu_scene *s, uint64_t paths, int sets) {
	if (paths <= s->cap_paths && sets <= s->wave_sets) return CRGPU_OK;
	if (s->wave.p) {
		cudaStreamSynchronize(s->stream);                           /* queued kernels may still use the old block */
		if (s->stream2) cudaStreamSynchronize(s->stream2);
	}
	s->cap_paths = 0; s->wave_sets = 0;
	const size_t n = ((size_t)paths + 255u) & ~(size_t)255u;      /* every sub-array stays 256-byte aligned */
	const size_t per_set = n * (9u * 16u + 2u * 4u + 1u);         /* 153 B per path */
	int rc = s->wave.alloc(s->device, per_set * (size_t)sets);
	if (rc) return rc;
	for (int k = 0; k < sets; ++k) {
		WaveBuffers &w = k ? s->wb2 : s->wb;
		uint8_t *q = s->wave.as<uint8_t>() + per_set * (size_t)k;
		auto take = [&](size_t b) { uint8_t *r = q; q += b; return r; };
		w.stA[0] = (float4 *)take(n * 16); w.stA[1] = (float4 *)take(n * 16);
		w.stB[0] = (float4 *)take(n * 16); w.stB[1] = (float4 *)take(n * 16);
		w.stC[0] = (uint4 *)take(n * 16); w.stC[1] = (uint4 *)take(n * 16);
		w.hit = (float4 *)take(n * 16); w.L = (float4 *)take(n * 16);
		w.hitInst = (int *)take(n * 4); w.perm = (unsigned *)take(n * 4);
		w.hitKey = (unsigned char *)take(n);
		w.perm2 = (unsigned *)take(n * 4); w.dirKey = (unsigned char *)take(n);
	}
	s->cap_paths = paths;
	s->wave_sets = sets;
	return CRGPU_OK;
}

extern "C" int crgpu_scene_destroy(crgpu_scene *s) {
	if (!s) return CRGPU_OK;
	cudaSetDevice(s->device);
	if (s->stream) cudaStreamSynchronize(s->stream);
	if (s->own_stream && s->own_stream != s->stream) cudaStreamSynchronize(s->own_stream);
	if (s->stream2) cudaStreamSynchronize(s->stream2);
	for (cudaEvent_t e : s->ev) if (e) cudaEventDestroy(e);
	for (cudaEvent_t e : s->evAcc) if (e) cudaEventDestroy(e);
	if (s->evFork) cudaEventDestroy(s->evFork);
	if (s->stream2) cudaStreamDestroy(s->stream2);
	if (s->own_stream) cudaStreamDestroy(s->own_stream);
	if (s->snap_stream) cudaStreamDestroy(s->snap_stream);
	if (s->stop_host) cudaFreeHost(s->stop_host);
	if (s->adapt_host) cudaFreeHost(s->adapt_host);
	delete s;                                        /* its blocks go back to the per-device cache */
	return CRGPU_OK;
}

extern "C" void crgpu_prepared_free(crgpu_prepared *p) {
	if (!p) return;
	if (p->slab) { if (p->pinned) cudaFreeHost(p->slab); else free(p->slab); }
	delete p;
}
static int pfail(crgpu_prepared *p, int rc) { crgpu_prepared_free(p); return rc; }

extern "C" int crgpu_prepared_update_config(crgpu_prepared *p, const struct crs_scene *f) {
	if (!p || !f) return fail(CRGPU_ERR_BAD_ARGUMENT, "NULL argument");
	if (f->prefs.image_width == 0 || f->prefs.image_height == 0 || f->prefs.sample_count == 0)
		return fail(CRGPU_ERR_BAD_ARGUMENT, "empty image or zero samples");
	p->prefs = f->prefs;
	p->camera = f->camera;
	return CRGPU_OK;
}

extern "C" int crgpu_prepared_materials(const crgpu_prepared *p, uint32_t *kinds, uint32_t *flags, uint32_t count, uint32_t *material_count) {
	if (!p || (count && (!kinds || !flags))) return fail(CRGPU_ERR_BAD_ARGUMENT, "NULL argument");
	const DevFlat *fl = reinterpret_cast<const DevFlat *>(p->slab + p->off[SEC_FLAT]);
	for (uint32_t i = 0; i < count && i < p->material_count; ++i) { kinds[i] = fl[i].kind; flags[i] = fl[i].flags; }
	if (material_count) *material_count = p->material_count;
	return CRGPU_OK;
}

extern "C" int crgpu_prepared_background(const crgpu_prepared *p, uint32_t *kind) {
	if (!p || !kind) return fail(CRGPU_ERR_BAD_ARGUMENT, "NULL argument");
	*kind = p->bg.kind;
	return CRGPU_OK;
}

extern "C" int crgpu_prepared_top_level(const crgpu_prepared *p, const void **items, size_t *item_bytes, const void **instances,
                                        size_t *instance_bytes, const void **bvhs, size_t *bvh_bytes) {
	if (!p || !items || !item_bytes || !instances || !instance_bytes || !bvhs || !bvh_bytes) return fail(CRGPU_ERR_BAD_ARGUMENT, "NULL argument");
	static_assert(sizeof(DevInstance) == 128 && sizeof(DevBvh) == 60, "crgpu_prepared_top_level documents these record sizes");
	*items = p->slab + p->off[SEC_TOP_ITEMS]; *item_bytes = p->len[SEC_TOP_ITEMS];
	*instances = p->slab + p->off[SEC_INSTS]; *instance_bytes = p->len[SEC_INSTS];
	*bvhs = p->slab + p->off[SEC_BVHS]; *bvh_bytes = p->len[SEC_BVHS];
	return CRGPU_OK;
}

extern "C" int crgpu_prepared_slab(const crgpu_prepared *p, const void **slab, size_t *bytes) {
	if (!p) return fail(CRGPU_ERR_BAD_ARGUMENT, "NULL argument");
	if (slab) *slab = p->slab;
	if (bytes) *bytes = p->slab_bytes;
	return CRGPU_OK;
}

extern "C" int crgpu_prepare(const struct crs_scene *f, crgpu_prepared **out) {
	if (!f || !out) return fail(CRGPU_ERR_BAD_ARGUMENT, "NULL argument");
	*out = nullptr;
	if (f->prefs.image_width == 0 || f->prefs.image_height == 0 || f->prefs.sample_count == 0)
		return fail(CRGPU_ERR_BAD_ARGUMENT, "empty image or zero samples");
	if (!node_ok(f, f->background) || f->nodes[f->background].kind != CRS_BSDF_BACKGROUND)
		return fail(CRGPU_ERR_UNSUPPORTED, "scene background must be a background node");
	if (f->top_bvh >= f->bvh_count) return fail(CRGPU_ERR_BAD_ARGUMENT, "top_bvh out of range");
	crgpu_prepared *p = new crgpu_prepared();
	p->slab = nullptr; p->pinned = false; p->slab_bytes = 0;
	p->prefs = f->prefs; p->camera = f->camera; p->background = f->background; p->instance_count = f->instance_count;
	p->texture_count = f->texture_count;
#define PFAIL(x) do { int rc_ = (x); if (rc_) return pfail(p, rc_); } while (0)

	/* materials, node graph, textures, background (their checks come before the geometry's: a scene malformed in both reports
	 * its shading error) */
	ShadingFold sh;
	PFAIL(fold_shading(f, sh));
	p->xnodes = sh.xnodes;
	p->bg = sh.bg;
	const std::vector<DevMaterial> &mats = sh.mats;
	const std::vector<DevFlat> &flat = sh.flat;
	const std::vector<DevTexture> &texs = sh.texs;
	const std::vector<uint8_t> &order = sh.order;
	p->flat_keys = sh.flat_keys;

	/* BVHs → pair nodes; triangles in leaf order; per-poly shading records.  The three products are independent once the
	 * slot offsets are known, and every element is computed from the flat scene alone, so they are filled by index on a
	 * few host threads (the upload bytes do not depend on the thread count).  This is most of crgpu_scene_create's time. */
	std::vector<PairNode> pairs;
	std::vector<DevBvh> bvhs(f->bvh_count);
	std::vector<PackedTri> tris;
	std::vector<uint32_t> slot_poly;
	std::vector<int32_t> top_prims;
	std::vector<uint32_t> mesh_of_bvh(f->bvh_count, 0xffffffffu);
	for (uint32_t m = 0; m < f->mesh_count; ++m) {
		if (f->meshes[m].bvh >= f->bvh_count) { return pfail(p, fail(CRGPU_ERR_BAD_ARGUMENT, "mesh bvh index out of range")); }
		mesh_of_bvh[f->meshes[m].bvh] = m;
	}
	std::vector<uint32_t> slot_off(f->bvh_count, 0u);      /* first triangle slot of every mesh BVH (0 for the top level) */
	uint64_t total_slots = 0;
	for (uint32_t b = 0; b < f->bvh_count; ++b) {
		const crs_bvh &src = f->bvhs[b];
		if ((uint64_t)src.node_offset + src.node_count > f->bvh_node_count || (uint64_t)src.prim_offset + src.prim_count > f->prim_index_count) {
			return pfail(p, fail(CRGPU_ERR_BAD_ARGUMENT, "bvh %u ranges out of bounds", b));
		}
		if (b == f->top_bvh) continue;
		if (mesh_of_bvh[b] == 0xffffffffu) { return pfail(p, fail(CRGPU_ERR_BAD_ARGUMENT, "bvh %u belongs to no mesh", b)); }
		slot_off[b] = (uint32_t)total_slots;
		total_slots += src.prim_count;
	}
	if (total_slots > 0xffffffffull) { return pfail(p, fail(CRGPU_ERR_UNSUPPORTED, "more than 2^32 triangle slots")); }
	for (uint32_t m = 0; m < f->mesh_count; ++m) {
		const crs_mesh &mesh = f->meshes[m];
		if ((uint64_t)mesh.poly_offset + mesh.poly_count > f->poly_count || (uint64_t)mesh.material_offset + mesh.material_count > f->material_count) {
			return pfail(p, fail(CRGPU_ERR_BAD_ARGUMENT, "mesh %u ranges out of bounds", m));
		}
	}
	tris.resize((size_t)total_slots);
	slot_poly.resize((size_t)total_slots);
	std::vector<ShadePoly> spolys(f->poly_count);
	HostError herr;

	/* (1) pair nodes of every BVH, in BVH order (sequential: each BVH appends behind the previous one) */
	std::thread pair_thread([&] {
		for (uint32_t b = 0; b < f->bvh_count; ++b) {
			const crs_bvh &src = f->bvhs[b];
			if (build_pairs(f, src, pairs, bvhs[b], b == f->top_bvh ? 0u : slot_off[b], &herr)) return;
			if (b != f->top_bvh) continue;
			for (uint32_t i = 0; i < src.prim_count; ++i) {
				const int32_t inst = f->prim_indices[src.prim_offset + i];
				if (inst < 0 || (uint32_t)inst >= f->instance_count) { herr.set(CRGPU_ERR_BAD_ARGUMENT, "top-level prim index out of range"); return; }
				top_prims.push_back(inst);
			}
		}
	});

	/* (2) triangles in leaf order */
	for (uint32_t b = 0; b < f->bvh_count; ++b) {
		if (b == f->top_bvh) continue;
		const crs_bvh &src = f->bvhs[b];
		const crs_mesh &mesh = f->meshes[mesh_of_bvh[b]];
		const uint32_t base = slot_off[b];
		host_parallel_for(src.prim_count, [&](uint32_t lo, uint32_t hi) {
			for (uint32_t i = lo; i < hi; ++i) {
				const int32_t local = f->prim_indices[src.prim_offset + i];
				if (local < 0 || (uint32_t)local >= mesh.poly_count) { herr.set(CRGPU_ERR_BAD_ARGUMENT, "prim index out of range"); return; }
				const uint32_t poly = mesh.poly_offset + (uint32_t)local;
				const crs_poly &p = f->polys[poly];
				for (int k = 0; k < 3; ++k)
					if (p.v[k] < 0 || (uint32_t)p.v[k] >= f->vertex_count) { herr.set(CRGPU_ERR_BAD_ARGUMENT, "vertex index out of range"); return; }
				float v0[3], v1[3], v2[3];
				f3(v0, f->vertices, (size_t)p.v[0]); f3(v1, f->vertices, (size_t)p.v[1]); f3(v2, f->vertices, (size_t)p.v[2]);
				PackedTri t;
				/* poly.c:20-22 — plain fp32 ops; this TU is compiled without contraction on the host side */
				for (int k = 0; k < 3; ++k) { t.v0[k] = v0[k]; t.e1[k] = v0[k] - v1[k]; t.e2[k] = v2[k] - v0[k]; }
				volatile float m0 = t.e1[1] * t.e2[2], m1 = t.e1[2] * t.e2[1], m2 = t.e1[2] * t.e2[0], m3 = t.e1[0] * t.e2[2],
							   m4 = t.e1[0] * t.e2[1], m5 = t.e1[1] * t.e2[0];
				t.n[0] = m0 - m1; t.n[1] = m2 - m3; t.n[2] = m4 - m5;
				tris[(size_t)base + i] = t;
				slot_poly[(size_t)base + i] = poly;
			}
		});
	}

	/* (3) per-poly shading records (meshes in order: should two meshes claim the same polygons, the later one wins as before) */
	for (uint32_t m = 0; m < f->mesh_count; ++m) {
		const crs_mesh &mesh = f->meshes[m];
		host_parallel_for(mesh.poly_count, [&](uint32_t lo, uint32_t hi) {
			for (uint32_t i = lo; i < hi; ++i) {
				const crs_poly &p = f->polys[mesh.poly_offset + i];
				ShadePoly sp;
				memset(&sp, 0, sizeof sp);
				bool has_n = p.has_normals != 0;
				for (int k = 0; k < 3 && has_n; ++k) if (p.n[k] < 0 || (uint32_t)p.n[k] >= f->normal_count) has_n = false;
				if (has_n) {
					f3(sp.n0, f->normals, (size_t)p.n[0]); f3(sp.n1, f->normals, (size_t)p.n[1]); f3(sp.n2, f->normals, (size_t)p.n[2]);
				} else if (p.has_normals) {
					herr.set(CRGPU_ERR_BAD_ARGUMENT, "normal index out of range"); return;
				} else {
					/* geometric normal e1 x e2 (poly.c:22,46), same operations as above */
					for (int k = 0; k < 3; ++k)
						if (p.v[k] < 0 || (uint32_t)p.v[k] >= f->vertex_count) { herr.set(CRGPU_ERR_BAD_ARGUMENT, "vertex index out of range"); return; }
					float v0[3], v1[3], v2[3], e1[3], e2[3];
					f3(v0, f->vertices, (size_t)p.v[0]); f3(v1, f->vertices, (size_t)p.v[1]); f3(v2, f->vertices, (size_t)p.v[2]);
					for (int k = 0; k < 3; ++k) { e1[k] = v0[k] - v1[k]; e2[k] = v2[k] - v0[k]; }
					volatile float m0 = e1[1] * e2[2], m1 = e1[2] * e2[1], m2 = e1[2] * e2[0], m3 = e1[0] * e2[2], m4 = e1[0] * e2[1], m5 = e1[1] * e2[0];
					sp.n0[0] = m0 - m1; sp.n0[1] = m2 - m3; sp.n0[2] = m4 - m5;
				}
				bool has_uv = mesh.texcoord_count != 0 && p.t[0] != -1;                          /* instance.c:151-153 */
				if (has_uv) {
					for (int k = 0; k < 3; ++k)
						if (p.t[k] < 0 || (uint32_t)p.t[k] >= f->texcoord_count) { herr.set(CRGPU_ERR_BAD_ARGUMENT, "texcoord index out of range"); return; }
					sp.t0[0] = f->texcoords[2 * (size_t)p.t[0]]; sp.t0[1] = f->texcoords[2 * (size_t)p.t[0] + 1];
					sp.t1[0] = f->texcoords[2 * (size_t)p.t[1]]; sp.t1[1] = f->texcoords[2 * (size_t)p.t[1] + 1];
					sp.t2[0] = f->texcoords[2 * (size_t)p.t[2]]; sp.t2[1] = f->texcoords[2 * (size_t)p.t[2] + 1];
				}
				if (p.material >= mesh.material_count) { herr.set(CRGPU_ERR_BAD_ARGUMENT, "poly material index out of range"); return; }
				sp.material = mesh.material_offset + p.material;
				sp.flags = (has_n ? 1u : 0u) | (has_uv ? 2u : 0u);
				spolys[mesh.poly_offset + i] = sp;
			}
		});
	}
	pair_thread.join();
	if (herr.code) { return pfail(p, fail(herr.code, "%s", herr.msg)); }

	/* instances */
	if (f->instance_count > CRG_ITEM_INDEX + 1u) { return pfail(p, fail(CRGPU_ERR_UNSUPPORTED, "more than 2^30 instances")); }
	InstancePack pk;
	PFAIL(pack_instances(f->instances, f->instance_count, f->spheres, f->sphere_count, f->meshes, f->mesh_count, f->material_count,
	                     CRGPU_ERR_UNSUPPORTED, pk));
	const std::vector<DevInstance> &insts = pk.recs;
	EditRecord &rec = p->rec;
	for (uint32_t i = 0; i < f->instance_count; ++i) {
		rec.inst_kind.push_back(f->instances[i].kind);
		rec.inst_object.push_back(f->instances[i].object);
	}
	rec.last = pk.last;
	rec.bvh_root.assign(6 * (size_t)f->bvh_count, 0.0f);
	for (uint32_t b = 0; b < f->bvh_count; ++b) {
		if (f->bvhs[b].node_count) memcpy(&rec.bvh_root[6 * (size_t)b], f->bvh_nodes[f->bvhs[b].node_offset].bounds, 6 * sizeof(float));
		rec.bvh_prims.push_back(f->bvhs[b].prim_count);
	}
	rec.meshes.assign(f->meshes, f->meshes + f->mesh_count);
	rec.spheres.assign(f->spheres, f->spheres + f->sphere_count);

	std::vector<crs_node> nodes(f->nodes, f->nodes + f->node_count);

	/* staging image: top-of-tree pair nodes (BFS prefix) of every BVH, the top level first, then the meshes
	 * in proportion to their size, CRG_STAGE_PAIRS nodes in total */
	std::vector<PairNode> stage;
	{
		auto take = [&](DevBvh &b, uint32_t quota) {
			const uint32_t internal = b.node_count > 1 ? (uint32_t)(b.pair_end - b.pair_offset) : 0u;
			const uint32_t cnt = quota < internal ? quota : internal;
			b.stage_base = (uint32_t)stage.size();
			b.stage_count = cnt;
			stage.insert(stage.end(), pairs.begin() + b.pair_offset, pairs.begin() + b.pair_offset + cnt);
		};
		/* shared memory and L1 share 228 KB per SM: every staged KB is a KB of L1 the traversal loses, so the default
		 * stages nothing; CRGPU_TRACE_STAGE=<pairs> (0..1024, read at every prepare) stages the top nodes of every BVH */
		const char *env = getenv("CRGPU_TRACE_STAGE");
		uint32_t total_budget = env ? (uint32_t)atoi(env) : 0u;
		if (total_budget > CRG_STAGE_PAIRS) total_budget = CRG_STAGE_PAIRS;
		take(bvhs[f->top_bvh], total_budget / 4);
		uint64_t total_internal = 0;
		for (uint32_t b = 0; b < f->bvh_count; ++b) if (b != f->top_bvh && bvhs[b].node_count > 1) total_internal += bvhs[b].pair_end - bvhs[b].pair_offset;
		const uint32_t budget = total_budget > (uint32_t)stage.size() ? total_budget - (uint32_t)stage.size() : 0u;
		for (uint32_t b = 0; b < f->bvh_count && total_internal; ++b) {
			if (b == f->top_bvh) continue;
			const uint64_t internal = bvhs[b].node_count > 1 ? bvhs[b].pair_end - bvhs[b].pair_offset : 0;
			take(bvhs[b], (uint32_t)((uint64_t)budget * internal / total_internal));
		}
	}
	p->top = bvhs[f->top_bvh];
	p->stage_pairs = (uint32_t)stage.size();
	/* the instance step's record of every top-level leaf item (the staging above has set every stage_count) */
	std::vector<DevTopItem> items(top_prims.size());
	for (size_t i = 0; i < top_prims.size(); ++i) items[i] = crg_top_item(insts[top_prims[i]], bvhs.data(), (uint32_t)top_prims[i]);
	{
		static const float unit[6] = { 0.f, 1.f, 0.f, 1.f, 0.f, 1.f };
		const crs_bvh &tb = f->bvhs[f->top_bvh];
		world_box(tb.node_count ? f->bvh_nodes[tb.node_offset].bounds : unit, p->world_lo, p->world_inv);
	}
	/* shading keys (K4's buckets): min(material + 1, 255) per prim slot from its poly, then per instance for spheres */
	std::vector<uint8_t> keys((size_t)total_slots + f->instance_count, 0u);
	host_parallel_for((uint32_t)total_slots, [&](uint32_t lo, uint32_t hi) {
		for (uint32_t i = lo; i < hi; ++i) keys[i] = shade_key(spolys[slot_poly[i]].material);
	});
	std::copy(pk.keys.begin(), pk.keys.end(), keys.begin() + (ptrdiff_t)total_slots);
	p->key_inst_off = (size_t)total_slots;
	p->material_count = f->material_count;
	std::vector<float> lut(256);
	for (int i = 0; i < 256; ++i) { volatile float num = (float)i, den = 255.0f; lut[i] = num / den; }   /* IEEE divss == __fdiv_rn */

	/* lay the sections out in one slab (256-byte aligned each) and copy them in on the host threads */
	const void *src[SEC_COUNT] = { stage.data(), pairs.data(), tris.data(), slot_poly.data(), keys.data(), spolys.data(), items.data(), bvhs.data(),
								   insts.data(), mats.data(), flat.data(), order.data(), nodes.data(), texs.data(), lut.data(), f->texdata };
	const size_t len[SEC_COUNT] = { stage.size() * sizeof(PairNode), pairs.size() * sizeof(PairNode), tris.size() * sizeof(PackedTri),
									slot_poly.size() * sizeof(uint32_t), keys.size(), spolys.size() * sizeof(ShadePoly), items.size() * sizeof(DevTopItem),
									bvhs.size() * sizeof(DevBvh), insts.size() * sizeof(DevInstance), mats.size() * sizeof(DevMaterial),
									flat.size() * sizeof(DevFlat), order.size(), nodes.size() * sizeof(crs_node), texs.size() * sizeof(DevTexture), lut.size() * sizeof(float), (size_t)f->texdata_bytes };
	size_t total = 0;
	for (int k = 0; k < SEC_COUNT; ++k) { p->off[k] = total; p->len[k] = len[k]; total += (len[k] + 255u) & ~(size_t)255u; }
	total += 512;                                                  /* room for the DevScene descriptor behind the arrays */
	p->slab_bytes = total;
	void *host = nullptr;
	if (cudaHostAlloc(&host, total, cudaHostAllocPortable) == cudaSuccess) p->pinned = true;
	else { cudaGetLastError(); host = malloc(total); p->pinned = false; }   /* no device yet (host-only tooling): pageable works, slower */
	if (!host) return pfail(p, fail(CRGPU_ERR_NOMEM, "cannot allocate the %zu-byte host slab", total));
	p->slab = static_cast<uint8_t *>(host);
	for (int k = 0; k < SEC_COUNT; ++k) {
		uint8_t *dst = p->slab + p->off[k];
		const uint8_t *from = static_cast<const uint8_t *>(src[k]);
		const size_t n = len[k];
		if (n) host_parallel_for((uint32_t)((n + 4095u) / 4096u), [&](uint32_t lo, uint32_t hi) {
			const size_t b0 = (size_t)lo * 4096u, b1 = (size_t)hi * 4096u < n ? (size_t)hi * 4096u : n;
			if (b1 > b0) memcpy(dst + b0, from + b0, b1 - b0);
		});
		memset(dst + n, 0, (((n + 255u) & ~(size_t)255u) - n));
	}
	memset(p->slab + total - 512, 0, 512);
#undef PFAIL
	*out = p;
	return CRGPU_OK;
}

extern "C" int crgpu_scene_create_prepared(const crgpu_prepared *p, int device, crgpu_scene **out) {
	if (!p || !out) return fail(CRGPU_ERR_BAD_ARGUMENT, "NULL argument");
	*out = nullptr;
	int ndev = 0;
	int rc = crgpu_device_count(&ndev);
	if (rc) return rc;
	if (device < 0 || device >= ndev) return fail(CRGPU_ERR_BAD_ARGUMENT, "device %d out of range (have %d)", device, ndev);
	CU(cudaSetDevice(device));

	crgpu_scene *s = new crgpu_scene();
	s->device = device; s->xnodes = p->xnodes;
	s->rec = p->rec;
	const DevBvh *bvhs = reinterpret_cast<const DevBvh *>(p->slab + p->off[SEC_BVHS]);
	s->bvhs.assign(bvhs, bvhs + p->len[SEC_BVHS] / sizeof(DevBvh));
	for (const DevBvh &b : s->bvhs) s->stage_cap.push_back(b.stage_count);
	s->mesh_region.assign(p->rec.meshes.size(), 0xffffffffu);
	s->pair_count = s->pair_cap = (uint32_t)(p->len[SEC_PAIRS] / sizeof(PairNode));
	s->top_off = s->pair_count;
	s->top_cap = p->instance_count > 1u ? p->instance_count - 1u : 1u;
	s->top_stage_cap = p->top.stage_count;
	s->material_count = s->mat_cap = p->material_count;
	s->slot_count = s->slot_cap = (uint32_t)p->key_inst_off;
	s->poly_count = s->poly_cap = (uint32_t)(p->len[SEC_SPOLYS] / sizeof(ShadePoly));
	s->bvh_cap = (uint32_t)s->bvhs.size();
#define FAIL_IF(x) do { int rc_ = (x); if (rc_) { crgpu_scene_destroy(s); return rc_; } } while (0)
#define CUS(call) do { cudaError_t e_ = (call); if (e_ != cudaSuccess) { int rc_ = fail(CRGPU_ERR_CUDA, "%s: %s", #call, cudaGetErrorString(e_)); crgpu_scene_destroy(s); return rc_; } } while (0)
	CUS(cudaDeviceGetAttribute(&s->sm_count, cudaDevAttrMultiProcessorCount, device));
	CUS(cudaStreamCreateWithFlags(&s->own_stream, cudaStreamNonBlocking));
	s->stream = s->own_stream;
	for (auto &e : s->ev) CUS(cudaEventCreate(&e));
	CUS(cudaStreamCreateWithFlags(&s->stream2, cudaStreamNonBlocking));
	for (auto &e : s->evAcc) CUS(cudaEventCreateWithFlags(&e, cudaEventDisableTiming));
	CUS(cudaEventCreateWithFlags(&s->evFork, cudaEventDisableTiming));

	/* the scene: one block, one copy */
	FAIL_IF(s->slab.alloc(device, p->slab_bytes));
	uint8_t *base = s->slab.as<uint8_t>();
	CUS(cudaMemcpyAsync(base, p->slab, p->slab_bytes, cudaMemcpyHostToDevice, s->stream));
	if (p->texture_count) {                 /* texture table with this device's addresses */
		std::vector<DevTexture> texs(p->texture_count);
		memcpy(texs.data(), p->slab + p->off[SEC_TEXS], p->texture_count * sizeof(DevTexture));
		for (DevTexture &t : texs) t.data = base + p->off[SEC_TEXDATA] + (uintptr_t)t.data;
		CUS(cudaMemcpyAsync(base + p->off[SEC_TEXS], texs.data(), texs.size() * sizeof(DevTexture), cudaMemcpyHostToDevice, s->stream));
		CUS(cudaStreamSynchronize(s->stream));   /* texs is a local pageable buffer */
	}
	DevScene &d = s->dev;
	d.cam = dev_camera(p->camera);
	d.image_width = p->prefs.image_width; d.image_height = p->prefs.image_height;
	d.sample_count = p->prefs.sample_count; d.bounces = p->prefs.bounces;
	d.background = p->background;
	d.instance_count = p->instance_count;
	d.top = p->top;
	d.stage_pairs = p->stage_pairs;
	memcpy(d.world_lo, p->world_lo, sizeof d.world_lo); memcpy(d.world_inv, p->world_inv, sizeof d.world_inv);
	d.stage_img = reinterpret_cast<const PairNode *>(base + p->off[SEC_STAGE]);
	d.pairs = reinterpret_cast<const PairNode *>(base + p->off[SEC_PAIRS]);
	d.tris = reinterpret_cast<const PackedTri *>(base + p->off[SEC_TRIS]);
	d.slot_poly = reinterpret_cast<const uint32_t *>(base + p->off[SEC_SLOT_POLY]);
	d.slot_key = reinterpret_cast<const uint8_t *>(base + p->off[SEC_KEYS]);
	d.inst_key = d.slot_key + p->key_inst_off;
	d.spolys = reinterpret_cast<const ShadePoly *>(base + p->off[SEC_SPOLYS]);
	d.top_items = reinterpret_cast<const DevTopItem *>(base + p->off[SEC_TOP_ITEMS]);
	d.bvhs = reinterpret_cast<const DevBvh *>(base + p->off[SEC_BVHS]);
	d.instances = reinterpret_cast<const DevInstance *>(base + p->off[SEC_INSTS]);
	d.materials = reinterpret_cast<const DevMaterial *>(base + p->off[SEC_MATS]);
	d.flat = reinterpret_cast<const DevFlat *>(base + p->off[SEC_FLAT]);
	d.key_order = base + p->off[SEC_ORDER];
	d.flat_keys = p->flat_keys;
	d.bg = p->bg;
	d.nodes = reinterpret_cast<const crs_node *>(base + p->off[SEC_NODES]);
	d.textures = reinterpret_cast<const DevTexture *>(base + p->off[SEC_TEXS]);
	d.u8_to_unit = reinterpret_cast<const float *>(base + p->off[SEC_LUT]);
	static_assert(sizeof(DevScene) <= 512, "DevScene must fit the descriptor slot behind the scene arrays");
	s->dev_copy = reinterpret_cast<DevScene *>(base + p->slab_bytes - 512);

	s->fb_floats = (size_t)d.image_width * d.image_height * 3u;
	FAIL_IF(s->fb.alloc(device, s->fb_floats * sizeof(float)));
	CUS(cudaMemsetAsync(s->fb.p, 0, s->fb.bytes, s->stream));
	{	/* per wave set: hist[1024] + counts[64] + box[CRG_BOX_SLOTS][12]; then the shared stats[80] and the stop words[16] */
		const size_t set_bytes = 1024 * sizeof(unsigned) + 256 + CRG_BOX_SLOTS * 12 * sizeof(unsigned);
		FAIL_IF(s->small.alloc(device, 2 * set_bytes + 80 * sizeof(unsigned long long) + 16 * sizeof(unsigned)));
		CUS(cudaMemsetAsync(s->small.p, 0, s->small.bytes, s->stream));
		uint8_t *sm = s->small.as<uint8_t>();
		s->wb.hist = reinterpret_cast<unsigned *>(sm);
		s->wb.counts = s->wb.hist + 1024;
		s->wb.box = s->wb.hist + 1024 + 64;
		s->wb2.hist = reinterpret_cast<unsigned *>(sm + set_bytes);
		s->wb2.counts = s->wb2.hist + 1024;
		s->wb2.box = s->wb2.hist + 1024 + 64;
		s->wb.stats = s->wb2.stats = reinterpret_cast<unsigned long long *>(sm + 2 * set_bytes);
		s->stop_ctl = reinterpret_cast<unsigned *>(sm + 2 * set_bytes + 80 * sizeof(unsigned long long));
	}
	{
		/* Paths in flight per wavefront batch.  Every batch pays a fixed ~7 ms (the serial chain of its bounces: each
		 * late bounce lasts as long as its slowest ray), so batches should be as large as memory allows:
		 * 153 B of wavefront state per path; use at most 40% of the free HBM (cached blocks count as free), capped at 256M paths. */
		size_t free_b = 0, total_b = 0;
		CUS(cudaMemGetInfo(&free_b, &total_b));
		free_b += ctx_cached_bytes(device);
		uint64_t fit = (uint64_t)((double)free_b * 0.40 / 153.0);
		if (fit > (256ull << 20)) fit = 256ull << 20;
		if (fit < (1ull << 20)) fit = 1ull << 20;
		s->max_paths = fit;
	}
	FAIL_IF(publish(s));
#undef FAIL_IF
#undef CUS
	*out = s;
	return CRGPU_OK;
}

extern "C" int crgpu_scene_create(const struct crs_scene *f, int device, crgpu_scene **out) {
	if (!f || !out) return fail(CRGPU_ERR_BAD_ARGUMENT, "NULL argument");
	*out = nullptr;
	int ndev = 0;
	int rc = crgpu_device_count(&ndev);
	if (rc) return rc;
	if (device < 0 || device >= ndev) return fail(CRGPU_ERR_BAD_ARGUMENT, "device %d out of range (have %d)", device, ndev);
	CU(cudaSetDevice(device));
	crgpu_prepared *p = nullptr;
	rc = crgpu_prepare(f, &p);
	if (rc) return rc;
	rc = crgpu_scene_create_prepared(p, device, out);
	crgpu_prepared_free(p);
	return rc;
}

extern "C" int crgpu_set_max_paths_in_flight(crgpu_scene *s, uint64_t max_paths) {
	if (!s || max_paths < 1024) return fail(CRGPU_ERR_BAD_ARGUMENT, "max_paths must be >= 1024");
	if (max_paths > (1ull << 31)) return fail(CRGPU_ERR_BAD_ARGUMENT, "max_paths must be <= 2^31");
	s->max_paths = max_paths;
	return CRGPU_OK;
}

static int check_rect(const crgpu_scene *s, int x0, int y0, int x1, int y1) {
	if (x0 < 0 || y0 < 0 || x1 > (int)s->dev.image_width || y1 > (int)s->dev.image_height || x1 <= x0 || y1 <= y0)
		return fail(CRGPU_ERR_BAD_ARGUMENT, "tile [%d,%d)x[%d,%d) outside the %ux%u image", x0, x1, y0, y1, s->dev.image_width, s->dev.image_height);
	return CRGPU_OK;
}

/* The gates of an armed call in one batch loop (render_batches); an unarmed call runs none.  A whole call: every batch checks the
 * stop word and publishes.  A piece of a pass-major walk (one batch of passes over one piece): only the first piece of a pass batch
 * checks the stop word, the later ones follow its decision, and the last piece publishes the pass batch. */
struct Gates {
	bool check;                /* reset the abandoned flag at the first gate and check the stop word at every gate */
	bool publish;              /* publish after K5 */
	bool whole;                /* a whole call: stop enqueueing batches once the stop word is set */
	uint64_t call_pixels;      /* pixels of the whole call (a pass batch commits call_pixels * passes paths) */
};
static bool stop_requested(const crgpu_scene *s) { return __atomic_load_n(&s->stop_host[0], __ATOMIC_ACQUIRE) != 0u; }

/* CRGPU_FLAG_TIME_KERNELS: events around the kernels of one batch loop.  Per batch K1's start and end (k1); per bounce TEV events
 * (bounce): before K2, after K2, after K4, after each of K3's miss / flat / generic launches, after the K4b sort. */
struct KernelTimes {
	enum { TEV = 7 };
	std::vector<cudaEvent_t> k1, bounce;
	static void mark(std::vector<cudaEvent_t> &v, cudaStream_t on) { cudaEvent_t e; cudaEventCreate(&e); cudaEventRecord(e, on); v.push_back(e); }
	~KernelTimes() {
		for (cudaEvent_t e : k1) cudaEventDestroy(e);
		for (cudaEvent_t e : bounce) cudaEventDestroy(e);
	}
	/* once the events have completed: add the loop's time (s->ev[0] .. s->ev[1]) and its K2 and K4 + K3 + K4b times to the scene's
	 * pending stats, and report them on stderr under CRGPU_DUMP_TIMES */
	void fold(crgpu_scene *s, int maxDepth) const {
		float total_ms = 0.f, trace_ms = 0.f, shade_ms = 0.f;
		cudaEventElapsedTime(&total_ms, s->ev[0], s->ev[1]);
		const char *dump = getenv("CRGPU_DUMP_TIMES");
		const int dump_level = dump ? atoi(dump) : 0;
		/* CRGPU_DUMP_TIMES=2: K1 per batch, and per bounce K2 (trace), K4 + K3 (shade) and shade's parts: K4, K3's miss / flat / generic
		 * launches (an unsplit K3 counts as miss), the rest (the K4b sort) */
		for (size_t i = 0; dump_level > 1 && i + 2 <= k1.size(); i += 2) {
			float g = 0.f;
			cudaEventElapsedTime(&g, k1[i], k1[i + 1]);
			fprintf(stderr, "crgpu: batch %zu k1 %.3f ms\n", i / 2, g);
		}
		for (size_t i = 0; i + TEV <= bounce.size(); i += TEV) {
			float t[TEV - 1] = {};
			for (int k = 0; k + 1 < TEV; ++k) cudaEventElapsedTime(&t[k], bounce[i + (size_t)k], bounce[i + (size_t)k + 1]);
			const float a = t[0], b = t[1] + t[2] + t[3] + t[4] + t[5];
			trace_ms += a; shade_ms += b;
			const size_t n = i / TEV;
			if (dump && (a > 5.f || b > 8.f || dump_level > 1))
				fprintf(stderr, "crgpu: batch %zu depth %zu trace %.3f ms shade %.3f ms k4 %.3f miss %.3f flat %.3f generic %.3f sort %.3f\n",
				        n / (size_t)maxDepth, n % (size_t)maxDepth, a, b, t[1], t[2], t[3], t[4], t[5]);
		}
		s->pend_trace_ms += trace_ms; s->pend_shade_ms += shade_ms; s->pend_total_ms += total_ms;
	}
};

/* One bounce over half `cur` of a wave set: K2, K4 (the flat materials' buckets first when K3 has a flat launch), K3, and K4b when a
 * sort mode is set and another bounce follows.  Returns the number of kernels it enqueued.  times: NULL, or the timing events. */
static uint64_t enqueue_bounce(const crgpu_scene *s, const WaveBuffers &wb, int cur, int depth, int maxDepth, int dirmode, bool count, bool sorted,
                               bool xnodes, const TraceKnobs &kn, const ShadeKnobs &sk, cudaStream_t st, KernelTimes *times) {
	const int grid = s->sm_count * 8;
	if (times) times->mark(times->bounce, st);
	crg_launch_trace(s->dev, wb, cur, count, sorted, kn, st);
	if (times) times->mark(times->bounce, st);
	if (crg_shade_flat_order(sk)) crg_launch_bucket(wb, cur, grid, s->dev.key_order, (int)s->dev.flat_keys, st);
	else crg_launch_bucket(wb, cur, grid, nullptr, 0, st);
	cudaEvent_t k3ev[3] = { nullptr, nullptr, nullptr };
	if (times) {
		times->mark(times->bounce, st);
		for (cudaEvent_t &e : k3ev) { cudaEventCreate(&e); times->bounce.push_back(e); }
	}
	const bool sort_next = dirmode != 0 && depth + 1 < maxDepth;
	uint64_t launches = 2 + (uint64_t)crg_launch_shade(s->dev_copy, wb, cur, depth, maxDepth, sort_next ? dirmode : 0, xnodes, s->dev.bg.kind != CRG_BG_NONE,
	                                                   grid, sk, st, times ? k3ev : nullptr);
	if (sort_next) {                                                               /* K4b: the next bounce's rays by direction bin */
		crg_launch_dirsort(wb, cur ^ 1, dirmode == 4 ? (depth < CRG_BOX_SLOTS ? depth : CRG_BOX_SLOTS - 1) : -1, grid, st);
		++launches;
	}
	if (times) times->mark(times->bounce, st);
	return launches;
}

/* The batch loop: passes [pass_begin, +pass_count) over one piece of at most max_paths pixels (pass_count > 0).  vd: NULL, or the
 * piece's views (a views call: K1 and K5 in their views instantiations). */
static int render_batches(crgpu_scene *s, const TileDesc &base, uint64_t tile_pixels, int pass_begin, int pass_count, unsigned flags, const Gates &gates,
                          const ViewDesc *vd, AdaptPix *adapt) {
	const bool armed = s->armed;
	const bool count = (flags & CRGPU_FLAG_COUNT) != 0;
	const bool timing = (flags & CRGPU_FLAG_TIME_KERNELS) != 0;
	/* Batches.  A batch pays a fixed cost of several ms: its bounces 5..12 hold too few rays to fill the SMs (132 on H100), and every bounce lasts
	 * as long as its slowest ray.  So (1) batches are as large as the path budget allows and of EQUAL size (a 987 + 13 split wastes
	 * a whole tail on 13 passes), and (2) with two or more batches the budget is split into two wave sets that run on two streams:
	 * the thin tail of one batch overlaps the fat first bounces of the next.  Only the accumulate step is ordered (the running
	 * average is taken in pass order, renderer.c:288-291): batch b's k_accumulate waits for batch b-1's.  CRGPU_OVERLAP=0 disables. */
	static const int overlap_on = [] { const char *e = getenv("CRGPU_OVERLAP"); return e ? atoi(e) : 1; }();
	uint64_t batch = s->max_paths / tile_pixels;
	if (batch < 1) batch = 1;
	int sets = 1;
	if (overlap_on && !timing && !count && batch < (uint64_t)pass_count && batch >= 2) { sets = 2; batch /= 2; }
	if (batch > (uint64_t)pass_count) batch = (uint64_t)pass_count;
	{
		const uint64_t nb = ((uint64_t)pass_count + batch - 1) / batch;
		if (nb > 0) batch = ((uint64_t)pass_count + nb - 1) / nb;   /* equal shares */
		if (batch < 1) batch = 1;
	}
	int rc = alloc_wave(s, tile_pixels * batch, sets);
	if (rc) return rc;

	const int maxDepth = (int)s->dev.bounces;
	const int grid = s->sm_count * 8;
	const int dirmode = crg_dir_mode();
	const TraceKnobs &knobs = crg_trace_knobs_env();
	const ShadeKnobs &sknobs = crg_shade_knobs_env();
	uint64_t launches = 0;
	KernelTimes times;
	if (timing) CU(cudaEventRecord(s->ev[0], s->stream));
	if (sets == 2) {                /* fork: the second stream starts behind whatever is queued on the first */
		CU(cudaEventRecord(s->evFork, s->stream));
		CU(cudaStreamWaitEvent(s->stream2, s->evFork, 0));
	}
	int bi = 0;
	for (int pb = pass_begin; pb < pass_begin + pass_count; pb += (int)batch, ++bi) {
		if (armed && gates.whole && stop_requested(s)) break;       /* its gates would abandon it anyway */
		const int set = sets == 2 ? (bi & 1) : 0;
		cudaStream_t st = set ? s->stream2 : s->stream;
		const WaveBuffers &wb = set ? s->wb2 : s->wb;
		TileDesc td = base;
		td.npix = (unsigned)tile_pixels;
		td.order = crg_path_order();
		td.pass_begin = pb;
		td.pass_count = (pass_begin + pass_count - pb) < (int)batch ? (pass_begin + pass_count - pb) : (int)batch;
		if (timing) times.mark(times.k1, st);
		crg_launch_generate(s->dev, wb, td, vd, grid, st); ++launches;
		if (timing) times.mark(times.k1, st);
		/* bounces == 0: pathTrace's loop never runs and every sample is black (pathtrace.c:34-36,59).  L is write-once by
		 * design (cr_add_radiance / cr_finish_path), so with no bounce nothing would write it: clear it here instead */
		if (maxDepth == 0) CU(cudaMemsetAsync(wb.L, 0, (size_t)tile_pixels * (size_t)td.pass_count * sizeof(float4), st));
		if (armed && maxDepth == 0) { crg_launch_stop_gate(wb.counts, 0, s->stop_ctl, set, s->stop_host, gates.check, gates.check, st); ++launches; }
		int cur = 0;
		for (int depth = 0; depth < maxDepth; ++depth) {
			if (armed) { crg_launch_stop_gate(wb.counts, cur, s->stop_ctl, set, s->stop_host, gates.check && depth == 0, gates.check, st); ++launches; }
			if (depth >= CRG_TAIL_FROM && !count) { crg_launch_tail(s->dev_copy, wb, cur, depth, maxDepth, s->xnodes, st); ++launches; }
			launches += enqueue_bounce(s, wb, cur, depth, maxDepth, dirmode, count, dirmode != 0 && depth > 0, s->xnodes, knobs, sknobs, st,
			                           timing ? &times : nullptr);
			cur ^= 1;
		}
		if (sets == 2 && bi > 0) CU(cudaStreamWaitEvent(st, s->evAcc[set ^ 1], 0));      /* pass order of the running average */
		crg_launch_accumulate(s->fb.as<float>(), wb.L, td, (int)s->dev.image_width, (int)s->dev.image_height, grid, st, armed ? s->stop_ctl : nullptr, set,
		                      armed && gates.publish ? s->stop_host : nullptr, vd, adapt); ++launches;
		if (armed && gates.publish) {       /* stages a snapshot when K5 found one requested (crgpu_request_snapshot) */
			crg_launch_stop_publish(s->stop_ctl, set, s->stop_host, td.pass_begin, td.pass_count, gates.call_pixels * (uint64_t)td.pass_count, wb.stats,
			                        s->fb.as<float>(), s->snap8.as<uint8_t>(), s->fb_floats, s->sm_count * 4, st);
			++launches;
		}
		if (sets == 2) CU(cudaEventRecord(s->evAcc[set], st));      /* after the publish step: the next K5 reads what it wrote */
	}
	if (sets == 2 && bi > 0) {      /* join: everything queued later on the scene's stream comes after both */
		CU(cudaStreamWaitEvent(s->stream, s->evAcc[(bi - 1) & 1], 0));
		if (bi > 1) CU(cudaStreamWaitEvent(s->stream, s->evAcc[bi & 1], 0));
	}
	cudaStream_t st = s->stream;
	if (timing) CU(cudaEventRecord(s->ev[1], st));
	CU(cudaGetLastError());
	if (!armed) s->pend_paths += tile_pixels * (uint64_t)pass_count;   /* an armed call counts what its publish steps committed */
	s->pend_launches += launches;
	if (timing) {
		CU(cudaStreamSynchronize(st));
		times.fold(s, maxDepth);
	}
	return CRGPU_OK;
}

/* A pixel set cut into pieces of at most max_paths pixels: rows of the rectangle, or ranges of the list, or of a views call's view-major
 * numbering (so a piece may hold several views, or part of one).  A set that fits is one piece. */
struct Piece { TileDesc td; uint64_t pixels; ViewDesc vd; };
static int split_pieces(const crgpu_scene *s, const TileDesc &base, uint64_t tile_pixels, const ViewDesc *vd, std::vector<Piece> &pieces) {
	const uint64_t most = s->max_paths;
	const ViewDesc none = {};
	if (tile_pixels <= most) { pieces.push_back({ base, tile_pixels, vd ? *vd : none }); return CRGPU_OK; }
	if (base.pixels) {
		for (uint64_t p0 = 0; p0 < tile_pixels; p0 += most) {
			Piece p = { base, tile_pixels - p0 < most ? tile_pixels - p0 : most, vd ? *vd : none };
			if (vd) p.vd.p0 = (unsigned)p0;
			else p.td.pixels = base.pixels + p0;
			pieces.push_back(p);
		}
		return CRGPU_OK;
	}
	const uint64_t rows = most / (uint64_t)base.tw;
	if (rows < 1) return fail(CRGPU_ERR_BAD_ARGUMENT, "tile is %d pixels wide > max paths in flight %llu", base.tw, (unsigned long long)most);
	for (int y = 0; y < base.th; y += (int)rows) {
		Piece p = { base, 0, none };
		p.td.y0 = base.y0 + y;
		p.td.th = base.th - y < (int)rows ? base.th - y : (int)rows;
		p.pixels = (uint64_t)p.td.tw * (uint64_t)p.td.th;
		pieces.push_back(p);
	}
	return CRGPU_OK;
}

/* A render call: passes [pass_begin, +pass_count) over a pixel set (a rectangle, or an explicit list).  Unarmed, the pieces are
 * walked piece-major: every pass of a piece, its batches overlapped on the two wave sets, before the next piece.  Armed, every batch
 * commits in pass order or not at all (Gates, k_accumulate<true>, k_stop_publish), so the framebuffer then holds exactly passes
 * [0, committed) and a later call for [committed, end) finishes it bit for bit; several pieces are walked pass-major, each batch of
 * passes over every piece, so that one pass count describes the set.  Only the first piece of a pass batch takes a stop (the later
 * ones complete a pass batch whose first piece was added), which bounds its latency by one pass batch over the whole set.
 * vd: NULL, or the views of a views call over its whole (view, pixel) set of tile_pixels pairs (crgpu_render_views).  adapt: NULL, or
 * the pixel records of an adaptive round, which K5 updates with every pass it adds (crgpu_adaptive_round). */
static int render_call(crgpu_scene *s, const TileDesc &base, uint64_t tile_pixels, int pass_begin, int pass_count, unsigned flags, struct crgpu_stats *stats,
                       const ViewDesc *vd = nullptr, AdaptPix *adapt = nullptr) {
	if (pass_begin < 0 || pass_count < 0 || (uint64_t)pass_begin + (uint64_t)pass_count > s->dev.sample_count)
		return fail(CRGPU_ERR_BAD_ARGUMENT, "passes [%d,%d) outside [0,%u)", pass_begin, pass_begin + pass_count, s->dev.sample_count);
	const bool armed = s->armed;
	if (armed && !s->snap8.p) {
		CU(cudaSetDevice(s->device));
		int arc = alloc_srgb8(s, s->snap8);
		if (arc) return arc;
	}
	if (armed) {
		__atomic_store_n(&s->stop_host[1], (unsigned)pass_begin, __ATOMIC_RELEASE);
		__atomic_store_n(&s->stop_host[2], 1u, __ATOMIC_RELEASE);
		crg_launch_stop_begin(s->stop_ctl, s->stop_host, pass_begin, s->stream);
	}
	std::vector<Piece> pieces;
	int rc = CRGPU_OK;
	if (pass_count > 0 && tile_pixels > 0) rc = split_pieces(s, base, tile_pixels, vd, pieces);   /* an empty call renders nothing */
	if (!armed || pieces.size() < 2) {
		for (size_t k = 0; rc == CRGPU_OK && k < pieces.size(); ++k)
			rc = render_batches(s, pieces[k].td, pieces[k].pixels, pass_begin, pass_count, flags, { true, true, true, tile_pixels }, vd ? &pieces[k].vd : nullptr,
			                    adapt);
	} else {
		uint64_t widest = 1;
		for (const Piece &p : pieces) widest = p.pixels > widest ? p.pixels : widest;
		const int passes = (int)(s->max_paths / widest < 1 ? 1 : s->max_paths / widest);   /* one batch per piece */
		for (int pb = pass_begin; rc == CRGPU_OK && pb < pass_begin + pass_count; pb += passes) {
			if (stop_requested(s)) break;
			const int n = pass_begin + pass_count - pb < passes ? pass_begin + pass_count - pb : passes;
			for (size_t k = 0; rc == CRGPU_OK && k < pieces.size(); ++k)
				rc = render_batches(s, pieces[k].td, pieces[k].pixels, pb, n, flags, { k == 0, k + 1 == pieces.size(), false, tile_pixels },
				                    vd ? &pieces[k].vd : nullptr, adapt);
		}
	}
	if (armed) {
		crg_launch_stop_end(s->stop_ctl, s->stop_host, s->stream);   /* also after a failed enqueue: the in-flight word must clear */
		s->pend_launches += 2;
	}
	if (rc) return rc;
	CU(cudaGetLastError());
	if (flags & CRGPU_FLAG_ASYNC) return CRGPU_OK;
	rc = crgpu_get_stats(s, stats);
	if (rc || !armed) return rc;
	return __atomic_load_n(&s->stop_host[1], __ATOMIC_ACQUIRE) < (unsigned)(pass_begin + pass_count) ? CRGPU_STOPPED : CRGPU_OK;
}

/* wait for the work queued on the scene's streams */
static int drain(crgpu_scene *s) {
	CU(cudaSetDevice(s->device));
	CU(cudaStreamSynchronize(s->stream));
	if (s->stream2) CU(cudaStreamSynchronize(s->stream2));   /* NULL would be the legacy default stream */
	return CRGPU_OK;
}

extern "C" int crgpu_stop_enable(crgpu_scene *s, int on) {
	if (!s) return fail(CRGPU_ERR_BAD_ARGUMENT, "scene is NULL");
	int rc = drain(s);                                            /* no call of the other mode may still be in flight */
	if (rc) return rc;
	if (on && !s->stop_host) {
		void *p = nullptr;
		CU(cudaHostAlloc(&p, 64, cudaHostAllocMapped | cudaHostAllocPortable));   /* unified addressing: the same pointer on the device */
		s->stop_host = static_cast<unsigned *>(p);
	}
	if (on && !s->snap_stream) CU(cudaStreamCreateWithFlags(&s->snap_stream, cudaStreamNonBlocking));
	if (on) for (int k = 0; k < 16; ++k) __atomic_store_n(&s->stop_host[k], 0u, __ATOMIC_RELEASE);
	s->armed = on != 0;
	return CRGPU_OK;
}

extern "C" int crgpu_request_stop(crgpu_scene *s) {
	if (!s || !s->armed) return fail(CRGPU_ERR_BAD_ARGUMENT, "scene is NULL or not armed (crgpu_stop_enable)");
	__atomic_store_n(&s->stop_host[0], 1u, __ATOMIC_RELEASE);
	return CRGPU_OK;
}

extern "C" int crgpu_clear_stop(crgpu_scene *s) {
	if (!s || !s->armed) return fail(CRGPU_ERR_BAD_ARGUMENT, "scene is NULL or not armed (crgpu_stop_enable)");
	__atomic_store_n(&s->stop_host[0], 0u, __ATOMIC_RELEASE);
	return CRGPU_OK;
}

extern "C" int crgpu_progress(crgpu_scene *s, int *passes_done, int *busy) {
	if (!s || !s->armed) return fail(CRGPU_ERR_BAD_ARGUMENT, "scene is NULL or not armed (crgpu_stop_enable)");
	if (passes_done) *passes_done = (int)__atomic_load_n(&s->stop_host[1], __ATOMIC_ACQUIRE);
	if (busy) *busy = (int)__atomic_load_n(&s->stop_host[2], __ATOMIC_ACQUIRE);
	return CRGPU_OK;
}

/* Snapshots: host word [3] goes 0 (idle) -> 1 (requested, by the host) -> 2 (staged, by a publish step) -> 0 (taken, by the host).
 * Only the host leaves 2, so the device never writes the staging buffer while crgpu_take_snapshot may be copying it. */
extern "C" int crgpu_request_snapshot(crgpu_scene *s) {
	if (!s || !s->armed) return fail(CRGPU_ERR_BAD_ARGUMENT, "scene is NULL or not armed (crgpu_stop_enable)");
	unsigned idle = 0u;                    /* a request already made, or an image staged and not yet taken, stays as it is */
	__atomic_compare_exchange_n(&s->stop_host[3], &idle, 1u, false, __ATOMIC_ACQ_REL, __ATOMIC_ACQUIRE);
	return CRGPU_OK;
}

extern "C" int crgpu_take_snapshot(crgpu_scene *s, uint8_t *host_rgb8, int *passes_done) {
	if (!s || !s->armed) return fail(CRGPU_ERR_BAD_ARGUMENT, "scene is NULL or not armed (crgpu_stop_enable)");
	if (!host_rgb8) return fail(CRGPU_ERR_BAD_ARGUMENT, "host_rgb8 is NULL");
	unsigned *w = s->stop_host;
	CU(cudaSetDevice(s->device));
	if (__atomic_load_n(&w[3], __ATOMIC_ACQUIRE) != 2u) {
		if (__atomic_load_n(&w[2], __ATOMIC_ACQUIRE) != 0u) return CRGPU_PENDING;
		/* no call in flight (k_stop_end clears the word after the call's last publish step): the framebuffer is the committed image */
		int rc = crgpu_framebuffer_to_srgb8(s, host_rgb8);
		if (rc) return rc;
		if (passes_done) *passes_done = (int)__atomic_load_n(&w[1], __ATOMIC_ACQUIRE);
		__atomic_store_n(&w[3], 0u, __ATOMIC_RELEASE);
		return CRGPU_OK;
	}
	CU(cudaMemcpyAsync(host_rgb8, s->snap8.p, s->fb_floats, cudaMemcpyDeviceToHost, s->snap_stream));
	CU(cudaStreamSynchronize(s->snap_stream));
	if (passes_done) *passes_done = (int)__atomic_load_n(&w[4], __ATOMIC_ACQUIRE);
	__atomic_store_n(&w[3], 0u, __ATOMIC_RELEASE);
	return CRGPU_OK;
}

/* ---- scene edits between renders --------------------------------------------------------------------------------------------------
 * One edit call's change to the scene (DESIGN §4 "Editing a resident scene"): a copy of the descriptor to edit, the blocks the call
 * has staged, each bound for the scene member it replaces, and the layout of the pairs and instance blocks after the call.  apply()
 * moves the staged blocks in, publishes the descriptor once and only then lets the replaced blocks go back to the per-device cache.
 * A call that returns before apply() releases what it staged and leaves the scene as it was. */
struct Edit {
	crgpu_scene *s;
	DevScene dev;
	uint32_t pair_cap, top_off, top_cap;     /* crgpu_scene's, after the call */
	InstParts ip;
	uint32_t inst_cap;
	struct Staged { DevBlock *dst; DevBlock blk; };
	std::deque<Staged> staged;               /* a deque: stage() hands out references that later stages keep valid */
	explicit Edit(crgpu_scene *sc)
		: s(sc), dev(sc->dev), pair_cap(sc->pair_cap), top_off(sc->top_off), top_cap(sc->top_cap), ip(sc->ip), inst_cap(sc->inst_cap) {}
	/* the empty block that replaces dst at apply(); staging dst again releases the block staged before */
	DevBlock &stage(DevBlock &dst) {
		for (Staged &b : staged) if (b.dst == &dst) { b.blk.release(); return b.blk; }
		staged.push_back({ &dst, DevBlock() });
		return staged.back().blk;
	}
	/* what dst holds after apply() */
	const DevBlock &next(const DevBlock &dst) const {
		for (const Staged &b : staged) if (b.dst == &dst) return b.blk;
		return dst;
	}
	int apply() {
		for (Staged &b : staged) std::swap(*b.dst, b.blk);
		std::swap(s->dev, dev);
		const int rc = publish(s);
		if (rc) {                                /* the scene keeps its blocks and descriptor */
			for (Staged &b : staged) std::swap(*b.dst, b.blk);
			std::swap(s->dev, dev);
			return rc;
		}
		s->pair_cap = pair_cap; s->top_off = top_off; s->top_cap = top_cap;
		s->ip = ip; s->inst_cap = inst_cap;
		return CRGPU_OK;                         /* the replaced blocks, now in `staged`, go when the edit does */
	}
};

extern "C" int crgpu_scene_set_camera(crgpu_scene *s, const struct crs_camera *cam) {
	if (!s || !cam) return fail(CRGPU_ERR_BAD_ARGUMENT, "NULL argument");
	if (cam->width != (int32_t)s->dev.image_width || cam->height != (int32_t)s->dev.image_height)
		return fail(CRGPU_ERR_BAD_ARGUMENT, "camera is %dx%d, the scene renders %ux%u", cam->width, cam->height, s->dev.image_width, s->dev.image_height);
	int rc = drain(s);
	if (rc) return rc;
	Edit e(s);
	e.dev.cam = dev_camera(*cam);
	return e.apply();
}

static size_t align256(size_t b) { return (b + 255u) & ~(size_t)255u; }

/* Pair nodes a BVH of n primitives may need: the room of a top region or of a mesh region. */
static uint32_t region_pairs(uint32_t n) { return n > 1u ? n - 1u : 1u; }

/* Parts of one device block, 256-byte aligned, in the order they are taken.  A layout runs twice: over base 0 to size the block,
 * then over the block. */
struct Carve {
	uintptr_t base;
	size_t bytes;
	template <class T> T *take(size_t count) { T *q = reinterpret_cast<T *>(base + bytes); bytes += align256(count * sizeof(T)); return q; }
};
/* Lays layout's parts out over blk.  When they need more than blk holds, blk first goes back to the per-device cache (nothing in it
 * may be read any more) and a large enough block takes its place. */
template <class F> static int carve(int device, DevBlock &blk, F layout) {
	Carve c = { 0, 0 };
	layout(c);
	if (c.bytes > blk.bytes) {
		int rc = blk.alloc(device, c.bytes);
		if (rc) return rc;
	}
	c = { reinterpret_cast<uintptr_t>(blk.p), 0 };
	layout(c);
	return CRGPU_OK;
}

/* The top-level build's part of an edit call's scratch: the BVH roots it reads, the instance boxes, centres and ray offsets, the new
 * instance records, and the new top level's pairs and primitive order, for n instances.  A list edit also stages its last-instance
 * table and instance keys there; the other edits point `last` at the instance block's table. */
struct TopParts {
	float *roots, *bb, *ctr, *offs;
	DevInstance *insts;
	PairNode *pairs;
	int32_t *prims;
	uint32_t *last;
	uint8_t *keys;
};
static TopParts take_top(Carve &c, size_t roots, uint32_t n, bool list = false) {
	TopParts t;
	t.roots = c.take<float>(roots);
	t.bb = c.take<float>(6 * (size_t)n); t.ctr = c.take<float>(3 * (size_t)n); t.offs = c.take<float>(n);
	t.insts = c.take<DevInstance>(n);
	t.pairs = c.take<PairNode>(region_pairs(n));
	t.prims = c.take<int32_t>(n);
	t.last = list ? c.take<uint32_t>(n) : nullptr;
	t.keys = list ? c.take<uint8_t>(n) : nullptr;
	return t;
}

/* The instance block's parts for cap instances; `own`: with the scene's own instance records and keys. */
static InstParts take_insts(Carve &c, uint32_t cap, bool own) {
	InstParts q;
	q.last = c.take<uint32_t>(cap);
	q.items = c.take<DevTopItem>(cap);
	q.recs = own ? c.take<DevInstance>(cap) : nullptr;
	q.keys = own ? c.take<uint8_t>(cap) : nullptr;
	return q;
}

/* The DevBvh record of a device build whose pairs sit at pair_offset; it stages at most stage_cap of them at stage_base. */
static DevBvh bvh_record(const CrgBuildResult &res, uint32_t pair_offset, uint32_t slot_offset, uint32_t stage_base, uint32_t stage_cap) {
	DevBvh b;
	memset(&b, 0, sizeof b);
	b.pair_offset = pair_offset;
	b.pair_end = pair_offset + res.pairs;
	b.node_count = res.node_count;
	b.slot_offset = slot_offset;
	if (res.node_count == 1u) { memcpy(b.root_bounds, res.bounds, sizeof b.root_bounds); b.root_first = res.root_first; b.root_count = res.root_count; }
	b.stage_base = stage_base;
	b.stage_count = res.pairs < stage_cap ? res.pairs : stage_cap;
	return b;
}

/* Stages a pairs block of `count` pair nodes that starts with a copy of the edit's current ones (the uploaded pairs until the first
 * geometry edit; unedited meshes' pair offsets do not move). */
static int reserve_pairs(Edit &e, uint32_t count) {
	DevBlock blk;
	int rc = blk.alloc(e.s->device, (size_t)count * sizeof(PairNode));
	if (rc) return rc;
	CU(cudaMemcpyAsync(blk.p, e.dev.pairs, (size_t)e.pair_cap * sizeof(PairNode), cudaMemcpyDeviceToDevice, e.s->stream));
	e.dev.pairs = blk.as<const PairNode>();
	e.pair_cap = count;
	e.stage(e.s->pairs) = std::move(blk);
	return CRGPU_OK;
}

/* The first instance or mesh edit of a scene with instances stages its instance block for the uploaded list: EditRecord::last, then
 * room for the top level's item records.  The slab's instance records and keys stay in use until a list edit. */
static int stage_insts(Edit &e) {
	crgpu_scene *s = e.s;
	if (s->insts.p) return CRGPU_OK;
	const uint32_t n = (uint32_t)s->rec.last.size();
	int rc = carve(s->device, e.stage(s->insts), [&](Carve &c) { e.ip = take_insts(c, n, false); });
	if (rc) return rc;
	CU(cudaMemcpyAsync(e.ip.last, s->rec.last.data(), (size_t)n * 4u, cudaMemcpyHostToDevice, s->stream));
	e.inst_cap = n;
	return CRGPU_OK;
}

/* Instance boxes, ray offsets and the top-level BVH of n instances into the scratch parts t, mesh boxes from t.roots.  The records
 * start from `from` (the scene's current ones), or from what t.insts already holds when it is NULL; A and Ainv from inst (device)
 * when it is not NULL.  The offsets follow t.last. */
static int build_top(crgpu_scene *s, uint32_t n, const DevInstance *from, const crs_instance *inst, const TopParts &t, void *build,
                     CrgBuildResult *res) {
	cudaStream_t st = s->stream;
	if (from && n) CU(cudaMemcpyAsync(t.insts, from, (size_t)n * sizeof(DevInstance), cudaMemcpyDeviceToDevice, st));
	crg_launch_instance_boxes(inst, t.insts, t.roots, t.last, n, t.bb, t.ctr, t.offs, st);
	CU(cudaGetLastError());
	int rc = crg_bvh_build_pairs(t.bb, t.ctr, n, build, st, t.pairs, t.prims, res);
	if (rc) return rc;
	if (res->levels > CRG_MAX_STACK) return fail(CRGPU_ERR_UNSUPPORTED, "BVH deeper than 64 levels");
	return CRGPU_OK;
}

/* Copies a built top level of n instances over the edit's instance records, top region, item records and staged prefix, and points
 * its descriptor at them.  The BVH records the items read, the instance block and the top region must already be in place. */
static int commit_top(Edit &e, uint32_t n, const TopParts &t, const CrgBuildResult &res) {
	cudaStream_t st = e.s->stream;
	const DevBvh top = bvh_record(res, e.top_off, 0u, e.dev.top.stage_base, e.s->top_stage_cap);
	if (n) CU(cudaMemcpyAsync(const_cast<DevInstance *>(e.dev.instances), t.insts, (size_t)n * sizeof(DevInstance), cudaMemcpyDeviceToDevice, st));
	if (res.pairs) CU(cudaMemcpyAsync(const_cast<PairNode *>(e.dev.pairs) + top.pair_offset, t.pairs, (size_t)res.pairs * sizeof(PairNode), cudaMemcpyDeviceToDevice, st));
	crg_launch_top_items(t.prims, t.insts, e.dev.bvhs, n, e.ip.items, st);
	CU(cudaGetLastError());
	if (top.stage_count)
		CU(cudaMemcpyAsync(const_cast<PairNode *>(e.dev.stage_img) + top.stage_base, t.pairs, (size_t)top.stage_count * sizeof(PairNode), cudaMemcpyDeviceToDevice, st));
	e.dev.top = top;
	e.dev.top_items = e.ip.items;
	static const float unit[6] = { 0.f, 1.f, 0.f, 1.f, 0.f, 1.f };  /* crgpu_prepare's box of an empty top level */
	world_box(res.node_count ? res.bounds : unit, e.dev.world_lo, e.dev.world_inv);
	return CRGPU_OK;
}

/* Instance boxes, ray offsets and the top-level BVH of the edited instances are computed on the device, into scratch; only once the
 * build has passed the upload's checks are they copied over the scene's instances, top region and staged prefix, and the top-level
 * item records rebuilt from them. */
extern "C" int crgpu_scene_set_instances(crgpu_scene *s, const struct crs_instance *inst, uint32_t count) {
	if (!s || !inst) return fail(CRGPU_ERR_BAD_ARGUMENT, "NULL argument");
	const uint32_t n = (uint32_t)s->rec.inst_kind.size();
	if (count != n) return fail(CRGPU_ERR_BAD_ARGUMENT, "%u instances given, the scene has %u", count, n);
	for (uint32_t i = 0; i < n; ++i)
		if (inst[i].kind != s->rec.inst_kind[i] || inst[i].object != s->rec.inst_object[i])
			return fail(CRGPU_ERR_BAD_ARGUMENT, "instance %u changes its kind or object", i);
	int rc = drain(s);
	if (rc) return rc;
	if (n == 0) return CRGPU_OK;
	Edit e(s);
	crs_instance *dinst = nullptr;
	TopParts t;
	void *build = nullptr;
	rc = carve(s->device, s->scratch, [&](Carve &c) { dinst = c.take<crs_instance>(n); t = take_top(c, s->rec.bvh_root.size(), n); build = c.take<uint8_t>(crg_bvh_scratch_bytes(n)); });
	if (!rc) rc = stage_insts(e);
	if (rc) return rc;
	t.last = e.ip.last;
	/* the roots in a copy of their own: packing them behind the caller's instances would cost a host copy of every instance */
	CU(cudaMemcpyAsync(dinst, inst, (size_t)n * sizeof(crs_instance), cudaMemcpyHostToDevice, s->stream));
	CU(cudaMemcpyAsync(t.roots, s->rec.bvh_root.data(), s->rec.bvh_root.size() * sizeof(float), cudaMemcpyHostToDevice, s->stream));
	CrgBuildResult res;
	rc = build_top(s, n, s->dev.instances, dinst, t, build, &res);
	if (!rc && !s->pairs.p) rc = reserve_pairs(e, s->top_off + s->top_cap);
	if (!rc) rc = commit_top(e, n, t, res);
	if (!rc) rc = e.apply();
	return rc;
}

/* ---- instance-list edits ------------------------------------------------------------------------------------------------------------
 * The new list is validated and packed on the host (pack_instances, as crgpu_prepare packs it), and its boxes, ray offsets and top level
 * are built on the device into scratch (stage_list).  Only once the build has passed the upload's checks are the blocks staged
 * (grow_list): the pairs block grows when the top region cannot hold a top level of the new count, and the instance block is replaced
 * when it has no records of its own or no room for the new count.  Then the records, keys, last table, top region, item records and
 * staged prefix are written (commit_list). */

/* Uploads the packed list of n instances and the BVH roots (6 floats per BVH) into the scratch parts t (take_top with `list`) and builds
 * their boxes, ray offsets and top level there.  Changes nothing the kernels read. */
static int stage_list(crgpu_scene *s, const InstancePack &pk, uint32_t n, const std::vector<float> &roots, const TopParts &t, void *build,
                      CrgBuildResult *res) {
	cudaStream_t st = s->stream;
	if (n) {
		CU(cudaMemcpyAsync(t.insts, pk.recs.data(), (size_t)n * sizeof(DevInstance), cudaMemcpyHostToDevice, st));
		CU(cudaMemcpyAsync(t.last, pk.last.data(), (size_t)n * 4u, cudaMemcpyHostToDevice, st));
		CU(cudaMemcpyAsync(t.keys, pk.keys.data(), n, cudaMemcpyHostToDevice, st));
	}
	CU(cudaMemcpyAsync(t.roots, roots.data(), roots.size() * sizeof(float), cudaMemcpyHostToDevice, st));
	return build_top(s, n, nullptr, nullptr, t, build, res);
}

/* Stages the top region and instance block a list of n instances needs. */
static int grow_list(Edit &e, uint32_t n) {
	crgpu_scene *s = e.s;
	/* the top region: the current one while it holds any top level of n instances (region_pairs(n)), else a new one behind every pair
	 * of the block; mesh regions never move.  A region that has to move grows by half at least, so that adding instances a few at a
	 * time does not leave a trail of abandoned regions. */
	const bool block = e.next(s->pairs).p != nullptr;
	if (region_pairs(n) > e.top_cap) {
		const uint64_t want = (uint64_t)e.top_cap + e.top_cap / 2u;
		e.top_cap = want > region_pairs(n) ? (uint32_t)want : region_pairs(n);
		if (block) e.top_off = e.pair_cap;                /* before the first geometry edit the reserved region is simply larger */
	}
	const uint64_t need = (uint64_t)e.top_off + e.top_cap;
	if (need > 0xffffffffull / sizeof(PairNode)) return fail(CRGPU_ERR_UNSUPPORTED, "instance list: more pair nodes than the scene can address");
	int rc;
	if (!block || need > e.pair_cap) {
		rc = reserve_pairs(e, (uint32_t)(need > e.pair_cap ? need : e.pair_cap));
		if (rc) return rc;
	}
	/* the instance block: kept while it has records of its own and room for n, else a new one (growing by half at least) */
	if (!e.ip.recs || n > e.inst_cap) {
		const uint64_t grown = (uint64_t)e.inst_cap + e.inst_cap / 2u;
		const uint32_t cap = e.ip.recs && grown > n ? (uint32_t)(grown < 4194304u ? grown : 4194304u) : n;
		rc = carve(s->device, e.stage(s->insts), [&](Carve &c) { e.ip = take_insts(c, cap, true); });
		if (rc) return rc;
		e.inst_cap = cap;
	}
	return CRGPU_OK;
}

/* Writes a built list of n instances (stage_list) and its top level into the blocks grow_list staged. */
static int commit_list(Edit &e, uint32_t n, const TopParts &t, const CrgBuildResult &res) {
	cudaStream_t st = e.s->stream;
	if (n) {
		CU(cudaMemcpyAsync(e.ip.last, t.last, (size_t)n * 4u, cudaMemcpyDeviceToDevice, st));
		CU(cudaMemcpyAsync(e.ip.keys, t.keys, n, cudaMemcpyDeviceToDevice, st));
	}
	e.dev.instances = e.ip.recs;
	e.dev.inst_key = e.ip.keys;
	e.dev.instance_count = n;
	return commit_top(e, n, t, res);
}

/* the host records of a committed list of n instances */
static void record_list(crgpu_scene *s, const crs_instance *inst, uint32_t n, const InstancePack &pk) {
	EditRecord &r = s->rec;
	r.inst_kind.resize(n);
	r.inst_object.resize(n);
	for (uint32_t i = 0; i < n; ++i) { r.inst_kind[i] = inst[i].kind; r.inst_object[i] = inst[i].object; }
	r.last = pk.last;
}

extern "C" int crgpu_scene_set_instance_list(crgpu_scene *s, const struct crs_instance *inst, uint32_t count) {
	if (!s || (count && !inst)) return fail(CRGPU_ERR_BAD_ARGUMENT, "NULL argument");
	if (count > 4194304u) return fail(CRGPU_ERR_UNSUPPORTED, "%u instances (the device builder's limit is 4194304)", count);
	InstancePack pk;
	int rc = pack_instances(inst, count, s->rec.spheres.data(), (uint32_t)s->rec.spheres.size(), s->rec.meshes.data(), (uint32_t)s->rec.meshes.size(),
	                        s->material_count, CRGPU_ERR_BAD_ARGUMENT, pk);
	if (rc) return rc;
	rc = drain(s);
	if (rc) return rc;
	const uint32_t n = count;
	Edit e(s);
	TopParts t;
	void *build = nullptr;
	rc = carve(s->device, s->scratch, [&](Carve &c) { t = take_top(c, s->rec.bvh_root.size(), n, true); build = c.take<uint8_t>(crg_bvh_scratch_bytes(n)); });
	CrgBuildResult res;
	if (!rc) rc = stage_list(s, pk, n, s->rec.bvh_root, t, build, &res);
	if (!rc) rc = grow_list(e, n);
	if (!rc) rc = commit_list(e, n, t, res);
	if (!rc) rc = e.apply();
	if (!rc) record_list(s, inst, n, pk);
	return rc;
}

/* ---- mesh edits ---------------------------------------------------------------------------------------------------------------------
 * What one listed mesh reads from the caller's flat scene: its polys and the index ranges of vertices, normals and texcoords they use
 * (checked as crgpu_prepare checks them), and its parts of the scratch: inputs and rebuilt records. */
struct MeshEdit {
	uint32_t mesh, bvh, n;
	uint32_t vlo, vhi, nlo, nhi, tlo, thi;          /* [lo, hi) index ranges; hi == lo: none */
	crs_poly *polys;
	float *verts, *norms, *uvs, *bb, *ctr;
	PairNode *pairs;
	int32_t *prims;
	PackedTri *tris;
	uint32_t *slot;
	uint8_t *keys;
	ShadePoly *spolys;
	CrgBuildResult res;
};

static int check_mesh_polys(const crs_scene *f, const crs_mesh &mesh, MeshEdit &e) {
	struct Range { uint32_t lo = 0xffffffffu, hi = 0u; void add(int32_t i) { if ((uint32_t)i < lo) lo = (uint32_t)i; if ((uint32_t)i + 1u > hi) hi = (uint32_t)i + 1u; } };
	HostError herr;
	std::mutex merge;
	Range V, N, T;
	host_parallel_for(mesh.poly_count, [&](uint32_t lo, uint32_t hi) {
		Range v, nn, t;
		for (uint32_t i = lo; i < hi; ++i) {
			const crs_poly &p = f->polys[mesh.poly_offset + i];
			for (int k = 0; k < 3; ++k) {
				if (p.v[k] < 0 || (uint32_t)p.v[k] >= f->vertex_count) { herr.set(CRGPU_ERR_BAD_ARGUMENT, "vertex index out of range"); return; }
				v.add(p.v[k]);
			}
			if (p.has_normals)
				for (int k = 0; k < 3; ++k) {
					if (p.n[k] < 0 || (uint32_t)p.n[k] >= f->normal_count) { herr.set(CRGPU_ERR_BAD_ARGUMENT, "normal index out of range"); return; }
					nn.add(p.n[k]);
				}
			if (mesh.texcoord_count != 0 && p.t[0] != -1)                                  /* instance.c:151-153 */
				for (int k = 0; k < 3; ++k) {
					if (p.t[k] < 0 || (uint32_t)p.t[k] >= f->texcoord_count) { herr.set(CRGPU_ERR_BAD_ARGUMENT, "texcoord index out of range"); return; }
					t.add(p.t[k]);
				}
			if (p.material >= mesh.material_count) { herr.set(CRGPU_ERR_BAD_ARGUMENT, "poly material index out of range"); return; }
		}
		std::lock_guard<std::mutex> g(merge);
		for (auto pr : { std::make_pair(&V, &v), std::make_pair(&N, &nn), std::make_pair(&T, &t) })
			if (pr.second->hi) { if (pr.second->lo < pr.first->lo) pr.first->lo = pr.second->lo; if (pr.second->hi > pr.first->hi) pr.first->hi = pr.second->hi; }
	});
	if (herr.code) return fail(herr.code, "%s", herr.msg);
	e.vlo = V.hi ? V.lo : 0u; e.vhi = V.hi ? V.hi : 0u;
	e.nlo = N.hi ? N.lo : 0u; e.nhi = N.hi ? N.hi : 0u;
	e.tlo = T.hi ? T.lo : 0u; e.thi = T.hi ? T.hi : 0u;
	return CRGPU_OK;
}

/* the fields of a mesh record that fix its topology: an edit keeps them */
static bool same_mesh(const crs_mesh &a, const crs_mesh &b) {
	return a.poly_offset == b.poly_offset && a.poly_count == b.poly_count && a.material_offset == b.material_offset &&
	       a.material_count == b.material_count && a.texcoord_count == b.texcoord_count && a.bvh == b.bvh;
}

/* a mesh build's inputs and records in an edit call's scratch */
static void take_mesh(Carve &c, MeshEdit &e) {
	e.polys = c.take<crs_poly>(e.n);
	e.verts = c.take<float>(3 * (size_t)(e.vhi - e.vlo)); e.norms = c.take<float>(3 * (size_t)(e.nhi - e.nlo)); e.uvs = c.take<float>(2 * (size_t)(e.thi - e.tlo));
	e.bb = c.take<float>(6 * (size_t)e.n); e.ctr = c.take<float>(3 * (size_t)e.n);
	e.pairs = c.take<PairNode>(region_pairs(e.n)); e.prims = c.take<int32_t>(e.n);
	e.tris = c.take<PackedTri>(e.n); e.slot = c.take<uint32_t>(e.n); e.keys = c.take<uint8_t>(e.n); e.spolys = c.take<ShadePoly>(e.n);
}

/* Each mesh's triangle boxes, BVH, triangles, slot records and shading records, built on the device into its scratch parts from the
 * polys and the record f gives it.  Changes nothing the kernels read. */
static int build_meshes(crgpu_scene *s, const crs_scene *f, std::vector<MeshEdit> &edits, void *build) {
	cudaStream_t st = s->stream;
	for (MeshEdit &e : edits) {
		const crs_mesh &mesh = f->meshes[e.mesh];
		CU(cudaMemcpyAsync(e.polys, f->polys + mesh.poly_offset, (size_t)e.n * sizeof(crs_poly), cudaMemcpyHostToDevice, st));
		CU(cudaMemcpyAsync(e.verts, f->vertices + 3 * (size_t)e.vlo, (size_t)(e.vhi - e.vlo) * 12u, cudaMemcpyHostToDevice, st));
		if (e.nhi > e.nlo) CU(cudaMemcpyAsync(e.norms, f->normals + 3 * (size_t)e.nlo, (size_t)(e.nhi - e.nlo) * 12u, cudaMemcpyHostToDevice, st));
		if (e.thi > e.tlo) CU(cudaMemcpyAsync(e.uvs, f->texcoords + 2 * (size_t)e.tlo, (size_t)(e.thi - e.tlo) * 8u, cudaMemcpyHostToDevice, st));
		crg_launch_poly_boxes(e.polys, e.verts, e.vlo, e.n, e.bb, e.ctr, st);
		CU(cudaGetLastError());
		int rc = crg_bvh_build_pairs(e.bb, e.ctr, e.n, build, st, e.pairs, e.prims, &e.res);
		if (rc) return rc;
		if (e.res.levels > CRG_MAX_STACK) return fail(CRGPU_ERR_UNSUPPORTED, "mesh %u: BVH deeper than 64 levels", e.mesh);
		const CrgMeshRepack r = { e.polys, e.verts, e.norms, e.uvs, e.vlo, e.nlo, e.tlo, e.n, mesh.poly_offset, mesh.material_offset, mesh.texcoord_count };
		crg_launch_mesh_repack(r, e.prims, e.tris, e.slot, e.keys, e.spolys, st);
		CU(cudaGetLastError());
	}
	return CRGPU_OK;
}

/* Gives each mesh of `edits` that has no region yet (region[mesh] == UINT32_MAX) its own region of pair nodes behind every pair of the
 * block, in one reserve_pairs; the first geometry edit also reserves the top region behind the uploaded pairs. */
static int reserve_regions(Edit &ed, std::vector<uint32_t> &region, const std::vector<MeshEdit> &edits) {
	const uint32_t first = ed.next(ed.s->pairs).p ? ed.pair_cap : ed.top_off + ed.top_cap;
	uint64_t add = 0;
	for (const MeshEdit &e : edits) if (region[e.mesh] == 0xffffffffu) add += region_pairs(e.n);
	if ((uint64_t)first + add > 0xffffffffull / sizeof(PairNode)) return fail(CRGPU_ERR_UNSUPPORTED, "mesh edit: more pair nodes than the scene can address");
	if (first + add <= ed.pair_cap) return CRGPU_OK;
	int rc = reserve_pairs(ed, first + (uint32_t)add);
	if (rc) return rc;
	uint32_t next = first;
	for (const MeshEdit &e : edits)
		if (region[e.mesh] == 0xffffffffu) { region[e.mesh] = next; next += region_pairs(e.n); }
	return CRGPU_OK;
}

/* The sections the kernels read by triangle slot (tris, slot_poly, slot_key), by global poly (spolys) and by BVH (bvhs).  The slab holds
 * them until crgpu_scene_add_objects first grows them; the geometry block then holds them in this order. */
struct GeomParts {
	PackedTri *tris;
	uint32_t *slot_poly;
	uint8_t *slot_key;
	ShadePoly *spolys;
	DevBvh *bvhs;
};
static GeomParts geom_live(const DevScene &d) {
	return { const_cast<PackedTri *>(d.tris), const_cast<uint32_t *>(d.slot_poly), const_cast<uint8_t *>(d.slot_key),
	         const_cast<ShadePoly *>(d.spolys), const_cast<DevBvh *>(d.bvhs) };
}

/* Copies a built mesh over its pair region in the edit's pairs, its slots from slot_offset and its polys from poly_offset in the
 * sections g. */
static int commit_mesh(const Edit &ed, const MeshEdit &e, const GeomParts &g, uint32_t region, uint32_t slot_offset, uint32_t poly_offset) {
	cudaStream_t st = ed.s->stream;
	if (e.res.pairs) CU(cudaMemcpyAsync(const_cast<PairNode *>(ed.dev.pairs) + region, e.pairs, (size_t)e.res.pairs * sizeof(PairNode), cudaMemcpyDeviceToDevice, st));
	CU(cudaMemcpyAsync(g.tris + slot_offset, e.tris, (size_t)e.n * sizeof(PackedTri), cudaMemcpyDeviceToDevice, st));
	CU(cudaMemcpyAsync(g.slot_poly + slot_offset, e.slot, (size_t)e.n * 4u, cudaMemcpyDeviceToDevice, st));
	CU(cudaMemcpyAsync(g.slot_key + slot_offset, e.keys, e.n, cudaMemcpyDeviceToDevice, st));
	CU(cudaMemcpyAsync(g.spolys + poly_offset, e.spolys, (size_t)e.n * sizeof(ShadePoly), cudaMemcpyDeviceToDevice, st));
	return CRGPU_OK;
}

/* Each listed mesh's triangle boxes, BVH, triangles, slot records and shading records, then the instances and the top level, are
 * rebuilt on the device into scratch; only once every build has passed the upload's checks are they copied over the scene. */
extern "C" int crgpu_scene_set_meshes(crgpu_scene *s, const struct crs_scene *flat, const uint32_t *meshes, uint32_t count) {
	if (!s || !flat || (count && !meshes)) return fail(CRGPU_ERR_BAD_ARGUMENT, "NULL argument");
	const uint32_t nm = (uint32_t)s->rec.meshes.size();
	std::vector<uint8_t> listed(nm, 0u);
	std::vector<MeshEdit> edits;
	for (uint32_t k = 0; k < count; ++k) {
		const uint32_t m = meshes[k];
		if (m >= nm || m >= flat->mesh_count) return fail(CRGPU_ERR_BAD_ARGUMENT, "mesh %u out of range (the scene has %u)", m, nm);
		if (listed[m]) return fail(CRGPU_ERR_BAD_ARGUMENT, "mesh %u listed twice", m);
		listed[m] = 1u;
		const crs_mesh &a = s->rec.meshes[m], &b = flat->meshes[m];
		if (!same_mesh(a, b))
			return fail(CRGPU_ERR_BAD_ARGUMENT, "mesh %u: its record differs from the uploaded one (the topology cannot change)", m);
		if (a.bvh >= s->rec.bvh_prims.size() || s->rec.bvh_prims[a.bvh] != a.poly_count)
			return fail(CRGPU_ERR_BAD_ARGUMENT, "mesh %u: its uploaded BVH does not cover exactly its polys", m);
		if ((uint64_t)b.poly_offset + b.poly_count > flat->poly_count) return fail(CRGPU_ERR_BAD_ARGUMENT, "mesh %u ranges out of bounds", m);
		if (a.poly_count > 4194304u) return fail(CRGPU_ERR_UNSUPPORTED, "mesh %u: %u polys (the device builder's limit is 4194304)", m, a.poly_count);
		MeshEdit e;
		memset(&e, 0, sizeof e);
		e.mesh = m; e.bvh = a.bvh; e.n = a.poly_count;
		int rc = check_mesh_polys(flat, b, e);
		if (rc) return rc;
		if (e.n) edits.push_back(e);
	}
	int rc = drain(s);
	if (rc) return rc;
	if (edits.empty()) return CRGPU_OK;

	/* the scratch: every listed mesh's inputs and records, the top level's parts, then the builder's scratch for the largest build */
	const uint32_t ninst = (uint32_t)s->rec.inst_kind.size();
	uint32_t nmax = ninst;
	for (const MeshEdit &e : edits) nmax = e.n > nmax ? e.n : nmax;
	Edit ed(s);
	TopParts t;
	void *build = nullptr;
	rc = carve(s->device, s->scratch, [&](Carve &c) {
		for (MeshEdit &e : edits) take_mesh(c, e);
		t = take_top(c, s->rec.bvh_root.size(), ninst);
		build = c.take<uint8_t>(crg_bvh_scratch_bytes(nmax));
	});
	if (rc) return rc;
	rc = build_meshes(s, flat, edits, build);
	if (rc) return rc;
	cudaStream_t st = s->stream;

	/* the top level over the new mesh roots */
	std::vector<float> roots = s->rec.bvh_root;
	for (const MeshEdit &e : edits) memcpy(&roots[6 * (size_t)e.bvh], e.res.bounds, 6 * sizeof(float));
	CrgBuildResult top;
	memset(&top, 0, sizeof top);
	if (ninst) {
		CU(cudaMemcpyAsync(t.roots, roots.data(), roots.size() * sizeof(float), cudaMemcpyHostToDevice, st));
		rc = stage_insts(ed);
		t.last = ed.ip.last;
		if (!rc) rc = build_top(s, ninst, s->dev.instances, nullptr, t, build, &top);
		if (rc) return rc;
	}
	std::vector<uint32_t> region = s->mesh_region;
	rc = reserve_regions(ed, region, edits);
	if (rc) return rc;

	/* each mesh's region, slot and poly ranges, BVH record and staged prefix, then the instances and the top level */
	const GeomParts g = geom_live(ed.dev);
	std::vector<DevBvh> bvhs = s->bvhs;
	for (const MeshEdit &e : edits) {
		DevBvh &b = bvhs[e.bvh];
		rc = commit_mesh(ed, e, g, region[e.mesh], b.slot_offset, s->rec.meshes[e.mesh].poly_offset);
		if (rc) return rc;
		b = bvh_record(e.res, region[e.mesh], b.slot_offset, b.stage_base, s->stage_cap[e.bvh]);
		CU(cudaMemcpyAsync(g.bvhs + e.bvh, &b, sizeof b, cudaMemcpyHostToDevice, st));
		if (b.stage_count)
			CU(cudaMemcpyAsync(const_cast<PairNode *>(ed.dev.stage_img) + b.stage_base, e.pairs, (size_t)b.stage_count * sizeof(PairNode), cudaMemcpyDeviceToDevice, st));
	}
	if (ninst && (rc = commit_top(ed, ninst, t, top))) return rc;
	if ((rc = ed.apply())) return rc;
	s->rec.bvh_root = roots;
	s->bvhs = bvhs;
	s->mesh_region = region;
	return CRGPU_OK;
}

/* ---- shading edits ------------------------------------------------------------------------------------------------------------------
 * The records whose size the material count fixes (materials, flat records, K4's key order) are rewritten in place; the node graph,
 * texture table and texel data, whose sizes may change, go into a new shading block that replaces the previous one.  Every check and
 * the fold run first and the block is filled before anything the kernels read changes. */
/* The node graph, texture table (with the block's addresses) and texel data of `flat` in a staged shading block, uploaded and waited
 * for, and the edit's descriptor pointed at them. */
static int upload_shading(Edit &e, const crs_scene *flat, ShadingFold &sh) {
	crgpu_scene *s = e.s;
	crs_node *nodes = nullptr;
	DevTexture *texs = nullptr;
	uint8_t *data = nullptr;
	int rc = carve(s->device, e.stage(s->shade), [&](Carve &c) { nodes = c.take<crs_node>(flat->node_count); texs = c.take<DevTexture>(sh.texs.size()); data = c.take<uint8_t>(flat->texdata_bytes); });
	if (rc) return rc;
	for (DevTexture &t : sh.texs) t.data = data + (uintptr_t)t.data;
	cudaStream_t st = s->stream;
	if (flat->node_count) CU(cudaMemcpyAsync(nodes, flat->nodes, (size_t)flat->node_count * sizeof(crs_node), cudaMemcpyHostToDevice, st));
	if (!sh.texs.empty()) CU(cudaMemcpyAsync(texs, sh.texs.data(), sh.texs.size() * sizeof(DevTexture), cudaMemcpyHostToDevice, st));
	if (flat->texdata_bytes) CU(cudaMemcpyAsync(data, flat->texdata, (size_t)flat->texdata_bytes, cudaMemcpyHostToDevice, st));
	CU(cudaStreamSynchronize(st));
	e.dev.nodes = nodes;
	e.dev.textures = texs;
	return CRGPU_OK;
}
/* Writes the fold's materials (flat->material_count of them), flat records and key order over the edit's dev.materials, dev.flat and
 * dev.key_order, and sets its background. */
static int commit_shading(Edit &e, const crs_scene *flat, const ShadingFold &sh) {
	cudaStream_t st = e.s->stream;
	const size_t nm = flat->material_count;
	if (nm) {
		CU(cudaMemcpyAsync(const_cast<DevMaterial *>(e.dev.materials), sh.mats.data(), nm * sizeof(DevMaterial), cudaMemcpyHostToDevice, st));
		CU(cudaMemcpyAsync(const_cast<DevFlat *>(e.dev.flat), sh.flat.data(), nm * sizeof(DevFlat), cudaMemcpyHostToDevice, st));
	}
	CU(cudaMemcpyAsync(const_cast<uint8_t *>(e.dev.key_order), sh.order.data(), sh.order.size(), cudaMemcpyHostToDevice, st));
	e.dev.bg = sh.bg;
	e.dev.flat_keys = sh.flat_keys;
	e.dev.background = flat->background;
	return CRGPU_OK;
}

extern "C" int crgpu_scene_set_shading(crgpu_scene *s, const struct crs_scene *flat) {
	if (!s || !flat) return fail(CRGPU_ERR_BAD_ARGUMENT, "NULL argument");
	if (flat->material_count != s->material_count)
		return fail(CRGPU_ERR_BAD_ARGUMENT, "%u materials given, the scene has %u", flat->material_count, s->material_count);
	ShadingFold sh;
	int rc = fold_shading(flat, sh);
	if (rc) return rc;
	rc = drain(s);
	if (rc) return rc;
	Edit e(s);
	rc = upload_shading(e, flat, sh);
	if (!rc) rc = commit_shading(e, flat, sh);
	if (!rc) rc = e.apply();
	if (!rc) s->xnodes = sh.xnodes;
	return rc;
}

/* ---- adding objects -----------------------------------------------------------------------------------------------------------------
 * The scene takes the objects, shading and instance list of a grown flat scene B whose first meshes and spheres are the scene's.  Every
 * check, the shading fold and the instance packing run on the host first; then each new mesh is built on the device and the top level
 * over B's list, all into scratch (build_meshes, stage_list).  Only then are the blocks grown: a new shading block, the geometry block
 * when B's slots, polys or BVHs outgrow it, the materials block when B's materials do, one reserve_pairs for the new meshes' regions,
 * and the top region and instance block as an instance-list edit grows them.  The new meshes' records and the grown BVH table are
 * written behind the existing ones, the descriptor is published once, and only then do the replaced blocks go back to the cache. */

/* The geometry block's parts for the given room (GeomParts). */
static GeomParts take_geom(Carve &c, uint32_t slots, uint32_t polys, uint32_t bvhs) {
	GeomParts g;
	g.tris = c.take<PackedTri>(slots);
	g.slot_poly = c.take<uint32_t>(slots);
	g.slot_key = c.take<uint8_t>(slots);
	g.spolys = c.take<ShadePoly>(polys);
	g.bvhs = c.take<DevBvh>(bvhs);
	return g;
}
/* room for `need` in a section that holds `cap`: at least half as much again, so that objects added one at a time do not copy the
 * section every time */
static uint32_t grown_cap(uint32_t cap, uint32_t need) {
	const uint64_t g = (uint64_t)cap + cap / 2u;
	return need <= cap ? cap : (g > need ? (uint32_t)(g < 0xffffffffull ? g : 0xffffffffull) : need);
}
/* The materials block's parts (dev.materials, dev.flat). */
struct MatParts {
	DevMaterial *mats;
	DevFlat *flat;
};

extern "C" int crgpu_scene_add_objects(crgpu_scene *s, const struct crs_scene *flat) {
	if (!s || !flat) return fail(CRGPU_ERR_BAD_ARGUMENT, "NULL argument");
	const crs_scene &B = *flat;
	const uint32_t M = (uint32_t)s->rec.meshes.size(), S = (uint32_t)s->rec.spheres.size(), P = s->poly_count;
	if (B.mesh_count < M || B.sphere_count < S)
		return fail(CRGPU_ERR_BAD_ARGUMENT, "%u meshes and %u spheres given, the scene has %u and %u", B.mesh_count, B.sphere_count, M, S);
	if (B.top_bvh >= B.bvh_count) return fail(CRGPU_ERR_BAD_ARGUMENT, "top_bvh out of range");
	if (B.poly_count < P) return fail(CRGPU_ERR_BAD_ARGUMENT, "%u polys given, the scene has %u", B.poly_count, P);
	std::vector<uint8_t> bvh_taken(B.bvh_count, 0u);
	auto take_bvh = [&](uint32_t m, uint32_t b) {
		if (b >= B.bvh_count || b == B.top_bvh || bvh_taken[b]) return fail(CRGPU_ERR_BAD_ARGUMENT, "mesh %u: bvh index %u out of range, the top level's or another mesh's", m, b);
		bvh_taken[b] = 1u;
		return CRGPU_OK;
	};
	int rc;
	for (uint32_t m = 0; m < M; ++m) {
		const crs_mesh &b = B.meshes[m];
		if (!same_mesh(s->rec.meshes[m], b)) return fail(CRGPU_ERR_BAD_ARGUMENT, "mesh %u: its record differs from the scene's", m);
		if ((uint64_t)b.material_offset + b.material_count > B.material_count) return fail(CRGPU_ERR_BAD_ARGUMENT, "mesh %u ranges out of bounds", m);
		if ((rc = take_bvh(m, b.bvh))) return rc;
	}
	for (uint32_t k = 0; k < S; ++k)
		if (memcmp(&s->rec.spheres[k].radius, &B.spheres[k].radius, sizeof(float)))
			return fail(CRGPU_ERR_BAD_ARGUMENT, "sphere %u: its radius differs from the scene's", k);
	/* the new meshes: checked as crgpu_prepare checks them; their polys lie behind the scene's, one range each */
	std::vector<MeshEdit> edits;
	std::vector<uint32_t> empty;                     /* BVHs of new meshes without polys (no build: an empty BVH) */
	std::vector<std::pair<uint32_t, uint32_t>> ranges;
	uint64_t slots = s->slot_count;
	for (uint32_t m = M; m < B.mesh_count; ++m) {
		const crs_mesh &b = B.meshes[m];
		if (b.poly_offset < P || (uint64_t)b.poly_offset + b.poly_count > B.poly_count || (uint64_t)b.material_offset + b.material_count > B.material_count)
			return fail(CRGPU_ERR_BAD_ARGUMENT, "mesh %u ranges out of bounds", m);
		if ((rc = take_bvh(m, b.bvh))) return rc;
		if (b.poly_count > 4194304u) return fail(CRGPU_ERR_UNSUPPORTED, "mesh %u: %u polys (the device builder's limit is 4194304)", m, b.poly_count);
		MeshEdit e;
		memset(&e, 0, sizeof e);
		e.mesh = m; e.bvh = b.bvh; e.n = b.poly_count;
		if ((rc = check_mesh_polys(flat, b, e))) return rc;
		if (e.n) { edits.push_back(e); ranges.push_back({ b.poly_offset, b.poly_count }); }
		else empty.push_back(b.bvh);
		slots += b.poly_count;
	}
	std::sort(ranges.begin(), ranges.end());
	for (size_t k = 1; k < ranges.size(); ++k)
		if ((uint64_t)ranges[k - 1].first + ranges[k - 1].second > ranges[k].first) return fail(CRGPU_ERR_BAD_ARGUMENT, "new meshes share polys");
	if (slots > 0xffffffffull) return fail(CRGPU_ERR_UNSUPPORTED, "more than 2^32 triangle slots");
	ShadingFold sh;
	if ((rc = fold_shading(flat, sh))) return rc;
	const uint32_t n = B.instance_count;
	if (n && !B.instances) return fail(CRGPU_ERR_BAD_ARGUMENT, "NULL instances");
	if (n > 4194304u) return fail(CRGPU_ERR_UNSUPPORTED, "%u instances (the device builder's limit is 4194304)", n);
	InstancePack pk;
	if ((rc = pack_instances(B.instances, n, B.spheres, B.sphere_count, B.meshes, B.mesh_count, B.material_count, CRGPU_ERR_BAD_ARGUMENT, pk))) return rc;
	if ((rc = drain(s))) return rc;
	Edit ed(s);

	/* build into scratch: the new meshes, in BVH order (a fresh load gives them slots in that order), then the top level */
	std::sort(edits.begin(), edits.end(), [](const MeshEdit &a, const MeshEdit &b) { return a.bvh < b.bvh; });
	uint32_t nmax = n;
	for (const MeshEdit &e : edits) nmax = e.n > nmax ? e.n : nmax;
	const size_t nroots = 6 * (size_t)B.bvh_count;
	TopParts t;
	void *build = nullptr;
	rc = carve(s->device, s->scratch, [&](Carve &c) {
		for (MeshEdit &e : edits) take_mesh(c, e);
		t = take_top(c, nroots, n, true);
		build = c.take<uint8_t>(crg_bvh_scratch_bytes(nmax));
	});
	if (!rc) rc = build_meshes(s, flat, edits, build);
	if (rc) return rc;
	/* the grown host records: the new meshes' roots and primitive counts; B's BVH indices name the device records from here on */
	std::vector<float> roots = s->rec.bvh_root;
	std::vector<uint32_t> prims = s->rec.bvh_prims, stage_cap = s->stage_cap;
	std::vector<DevBvh> bvhs = s->bvhs;
	roots.resize(nroots, 0.f);
	prims.resize(B.bvh_count, 0u);
	stage_cap.resize(B.bvh_count, 0u);
	bvhs.resize(B.bvh_count);
	for (uint32_t b : empty) {
		memset(&bvhs[b], 0, sizeof(DevBvh));
		memset(&roots[6 * (size_t)b], 0, 6 * sizeof(float));
		prims[b] = 0u; stage_cap[b] = 0u;
	}
	for (const MeshEdit &e : edits) { memcpy(&roots[6 * (size_t)e.bvh], e.res.bounds, 6 * sizeof(float)); prims[e.bvh] = e.n; stage_cap[e.bvh] = 0u; }
	CrgBuildResult top;
	if ((rc = stage_list(s, pk, n, roots, t, build, &top))) return rc;

	/* stage: shading block, geometry block, materials block, the new meshes' pair regions, the list's top region and instance block */
	cudaStream_t st = s->stream;
	if ((rc = upload_shading(ed, flat, sh))) return rc;
	GeomParts g = geom_live(ed.dev);
	const uint32_t slot_need = (uint32_t)slots;
	uint32_t slot_cap = s->slot_cap, poly_cap = s->poly_cap, bvh_cap = s->bvh_cap;
	const bool grow_geom = slot_need > slot_cap || B.poly_count > poly_cap || B.bvh_count > bvh_cap;
	if (grow_geom) {
		slot_cap = grown_cap(slot_cap, slot_need); poly_cap = grown_cap(poly_cap, B.poly_count); bvh_cap = grown_cap(bvh_cap, B.bvh_count);
		if ((rc = carve(s->device, ed.stage(s->geom), [&](Carve &c) { g = take_geom(c, slot_cap, poly_cap, bvh_cap); }))) return rc;
		const GeomParts live = geom_live(s->dev);
		const size_t ns = s->slot_count;
		CU(cudaMemcpyAsync(g.tris, live.tris, ns * sizeof(PackedTri), cudaMemcpyDeviceToDevice, st));
		CU(cudaMemcpyAsync(g.slot_poly, live.slot_poly, ns * 4u, cudaMemcpyDeviceToDevice, st));
		CU(cudaMemcpyAsync(g.slot_key, live.slot_key, ns, cudaMemcpyDeviceToDevice, st));
		CU(cudaMemcpyAsync(g.spolys, live.spolys, (size_t)s->poly_count * sizeof(ShadePoly), cudaMemcpyDeviceToDevice, st));
	}
	const bool grow_mats = B.material_count > s->mat_cap;
	MatParts mp = { const_cast<DevMaterial *>(s->dev.materials), const_cast<DevFlat *>(s->dev.flat) };
	if (grow_mats &&
	    (rc = carve(s->device, ed.stage(s->mats), [&](Carve &c) { mp.mats = c.take<DevMaterial>(B.material_count); mp.flat = c.take<DevFlat>(B.material_count); })))
		return rc;
	std::vector<uint32_t> region = s->mesh_region;
	region.resize(B.mesh_count, 0xffffffffu);
	if ((rc = reserve_regions(ed, region, edits)) || (rc = grow_list(ed, n))) return rc;

	/* write: the new meshes and the BVH records (the list's item records read them), the shading, then the list and its top level */
	uint32_t slot = s->slot_count;
	for (const MeshEdit &e : edits) {
		if ((rc = commit_mesh(ed, e, g, region[e.mesh], slot, B.meshes[e.mesh].poly_offset))) return rc;
		bvhs[e.bvh] = bvh_record(e.res, region[e.mesh], slot, 0u, 0u);
		slot += e.n;
	}
	CU(cudaMemcpyAsync(g.bvhs, bvhs.data(), bvhs.size() * sizeof(DevBvh), cudaMemcpyHostToDevice, st));
	ed.dev.tris = g.tris; ed.dev.slot_poly = g.slot_poly; ed.dev.slot_key = g.slot_key; ed.dev.spolys = g.spolys; ed.dev.bvhs = g.bvhs;
	ed.dev.materials = mp.mats; ed.dev.flat = mp.flat;
	if ((rc = commit_shading(ed, flat, sh)) || (rc = commit_list(ed, n, t, top)) || (rc = ed.apply())) return rc;
	if (grow_geom) { s->slot_cap = slot_cap; s->poly_cap = poly_cap; s->bvh_cap = bvh_cap; }
	if (grow_mats) s->mat_cap = B.material_count;
	s->xnodes = sh.xnodes;
	record_list(s, B.instances, n, pk);
	s->material_count = B.material_count;
	s->slot_count = slot_need;
	s->poly_count = B.poly_count;
	s->mesh_region = region;
	s->bvhs = bvhs;
	s->stage_cap = stage_cap;
	EditRecord &r = s->rec;
	r.meshes.assign(B.meshes, B.meshes + B.mesh_count);
	r.spheres.assign(B.spheres, B.spheres + B.sphere_count);
	r.bvh_root = roots;
	r.bvh_prims = prims;
	return CRGPU_OK;
}

extern "C" int crgpu_scene_shading(crgpu_scene *s, uint32_t *kinds, uint32_t *flags, uint32_t count, uint32_t *material_count,
                                   uint32_t *background_kind, int *complete_interpreter) {
	if (!s || (count && (!kinds || !flags))) return fail(CRGPU_ERR_BAD_ARGUMENT, "NULL argument");
	const uint32_t n = count < s->material_count ? count : s->material_count;
	if (n) {
		int rc = drain(s);
		if (rc) return rc;
		std::vector<DevFlat> fl(n);
		CU(cudaMemcpyAsync(fl.data(), s->dev.flat, (size_t)n * sizeof(DevFlat), cudaMemcpyDeviceToHost, s->stream));
		CU(cudaStreamSynchronize(s->stream));
		for (uint32_t i = 0; i < n; ++i) { kinds[i] = fl[i].kind; flags[i] = fl[i].flags; }
	}
	if (material_count) *material_count = s->material_count;
	if (background_kind) *background_kind = s->dev.bg.kind;
	if (complete_interpreter) *complete_interpreter = s->xnodes ? 1 : 0;
	return CRGPU_OK;
}

extern "C" int crgpu_render_tile(crgpu_scene *s, int x0, int y0, int x1, int y1, int pass_begin, int pass_count,
								 unsigned flags, struct crgpu_stats *stats) {
	if (!s) return fail(CRGPU_ERR_BAD_ARGUMENT, "scene is NULL");
	int rc = check_rect(s, x0, y0, x1, y1);
	if (rc) return rc;
	CU(cudaSetDevice(s->device));
	TileDesc td;
	memset(&td, 0, sizeof td);
	td.x0 = x0; td.y0 = y0; td.tw = x1 - x0; td.th = y1 - y0;
	td.pixels = nullptr;
	return render_call(s, td, (uint64_t)td.tw * (uint64_t)td.th, pass_begin, pass_count, flags, stats);
}

/* The device pixel list of a tile set (rects = 4 ints per tile), built on the device and kept for the next call with the same set.
 * views: the view count of a views call, whose (view, pixel) pairs must number at most 2^32 - 1; 0 for crgpu_render_tiles. */
static int tile_set(crgpu_scene *s, const int *rects, int nrects, uint64_t views, uint64_t *total_out) {
	if (!rects || nrects < 1) return fail(CRGPU_ERR_BAD_ARGUMENT, "bad tile list");
	if (s->dev.image_width > 65535u || s->dev.image_height > 65535u) return fail(CRGPU_ERR_UNSUPPORTED, "tile lists need image dimensions <= 65535");
	CU(cudaSetDevice(s->device));
	uint64_t total = 0;
	for (int i = 0; i < nrects; ++i) {
		int rc = check_rect(s, rects[4 * i], rects[4 * i + 1], rects[4 * i + 2], rects[4 * i + 3]);
		if (rc) return rc;
		total += (uint64_t)(rects[4 * i + 2] - rects[4 * i]) * (uint64_t)(rects[4 * i + 3] - rects[4 * i + 1]);
	}
	if (views && total * views > 0xffffffffull)
		return fail(CRGPU_ERR_BAD_ARGUMENT, "%llu views of %llu pixels are more than 2^32 - 1 (view, pixel) pairs", (unsigned long long)views,
		            (unsigned long long)total);
	*total_out = total;
	std::vector<int> key(rects, rects + 4 * (size_t)nrects);
	if (key != s->pixel_key) {                         /* rebuild the pixel list only when the tile set changes */
		if (total > 0xffffffffull) return fail(CRGPU_ERR_UNSUPPORTED, "tile set of more than 2^32 pixels");
		/* the list is expanded ON THE DEVICE from the rectangles (a 1080p frame is 2 M entries, an 8K frame 33 M: building and
		 * uploading them from the host cost ~10 ms per frame): upload 16 B + 4 B per tile, one kernel writes x | y << 16 */
		std::vector<unsigned> offs((size_t)nrects);
		unsigned acc = 0u;
		for (int i = 0; i < nrects; ++i) { offs[(size_t)i] = acc; acc += (unsigned)((rects[4 * i + 2] - rects[4 * i]) * (rects[4 * i + 3] - rects[4 * i + 1])); }
		const size_t need = (size_t)total * sizeof(uint32_t) + (size_t)nrects * 20u + 256u;
		if (s->pixels.bytes < need) {
			CU(cudaStreamSynchronize(s->stream));       /* the previous list may still be in use by queued kernels */
			int arc = s->pixels.alloc(s->device, need);
			if (arc) return arc;
		}
		/* rectangle table behind the pixel list (same block); both copies are from pageable memory, i.e. staged before the call
		 * returns, and ordered before the kernel on the scene's stream */
		uint8_t *tab = s->pixels.as<uint8_t>() + (((size_t)total * sizeof(uint32_t) + 255u) & ~(size_t)255u);
		CU(cudaMemcpyAsync(tab, rects, (size_t)nrects * 16u, cudaMemcpyHostToDevice, s->stream));
		CU(cudaMemcpyAsync(tab + (size_t)nrects * 16u, offs.data(), (size_t)nrects * 4u, cudaMemcpyHostToDevice, s->stream));
		CU(cudaStreamSynchronize(s->stream));           /* offs is a local; costs ~20 us, once per tile set */
		crg_launch_pixel_list(s->pixels.as<uint32_t>(), reinterpret_cast<const int4 *>(tab), reinterpret_cast<const unsigned *>(tab + (size_t)nrects * 16u), nrects,
		                      crg_path_order().blocked, s->stream);
		CU(cudaGetLastError());
		s->pixel_key.swap(key);
	}
	return CRGPU_OK;
}

extern "C" int crgpu_render_tiles(crgpu_scene *s, const int *rects, int nrects, int pass_begin, int pass_count,
								  unsigned flags, struct crgpu_stats *stats) {
	if (!s) return fail(CRGPU_ERR_BAD_ARGUMENT, "bad tile list");
	uint64_t total = 0;
	int rc = tile_set(s, rects, nrects, 0, &total);
	if (rc) return rc;
	TileDesc td;
	memset(&td, 0, sizeof td);
	td.pixels = s->pixels.as<uint32_t>();
	return render_call(s, td, total, pass_begin, pass_count, flags, stats);
}

/* ---- several views in one call ---------------------------------------------------------------------------------------------------
 * The views block holds view_cap - 1 cameras, then view_cap - 1 framebuffers of fb_floats each (views 1 .. view_cap - 1). */
static size_t views_cam_bytes(uint32_t cap) { return align256((size_t)(cap - 1u) * sizeof(DevCamera)); }
static size_t views_bytes(uint32_t cap, size_t fb_floats) { return views_cam_bytes(cap) + (size_t)(cap - 1u) * fb_floats * sizeof(float); }
static float *views_fb(const DevBlock &b, uint32_t cap) { return b.p ? reinterpret_cast<float *>(static_cast<uint8_t *>(b.p) + views_cam_bytes(cap)) : nullptr; }
static float *view_fb(const crgpu_scene *s, uint32_t v) { return v ? views_fb(s->views, s->view_cap) + (size_t)(v - 1u) * s->fb_floats : s->fb.as<float>(); }

extern "C" int crgpu_scene_set_views(crgpu_scene *s, const struct crs_camera *cams, uint32_t count) {
	if (!s || !cams) return fail(CRGPU_ERR_BAD_ARGUMENT, "NULL argument");
	if (count < 1 || count > CRGPU_MAX_VIEWS) return fail(CRGPU_ERR_BAD_ARGUMENT, "%u views: the list holds 1 to %u", count, (unsigned)CRGPU_MAX_VIEWS);
	for (uint32_t i = 0; i < count; ++i)
		if (cams[i].width != (int32_t)s->dev.image_width || cams[i].height != (int32_t)s->dev.image_height)
			return fail(CRGPU_ERR_BAD_ARGUMENT, "camera %u is %dx%d, the scene renders %ux%u", i, cams[i].width, cams[i].height, s->dev.image_width,
			            s->dev.image_height);
	int rc = drain(s);
	if (rc) return rc;
	std::vector<DevCamera> dc(count - 1u);
	for (uint32_t i = 1; i < count; ++i) dc[i - 1u] = dev_camera(cams[i]);
	Edit e(s);
	const bool grow = count > s->view_cap;               /* a larger block; the surviving views' framebuffers move into it */
	const uint32_t cap = grow ? count : s->view_cap;
	if (grow && (rc = e.stage(s->views).alloc(s->device, views_bytes(cap, s->fb_floats)))) return rc;
	const DevBlock &blk = e.next(s->views);
	const uint32_t keep = s->view_count < count ? s->view_count : count;     /* views 0 .. keep - 1 keep their pixels */
	float *fbs = views_fb(blk, cap);
	const size_t fb_bytes = s->fb_floats * sizeof(float);
	cudaStream_t st = s->stream;
	if (grow && keep > 1u) CU(cudaMemcpyAsync(fbs, views_fb(s->views, s->view_cap), (size_t)(keep - 1u) * fb_bytes, cudaMemcpyDeviceToDevice, st));
	if (count > keep) CU(cudaMemsetAsync(fbs + (size_t)(keep - 1u) * s->fb_floats, 0, (size_t)(count - keep) * fb_bytes, st));
	if (count > 1u) CU(cudaMemcpyAsync(blk.p, dc.data(), dc.size() * sizeof(DevCamera), cudaMemcpyHostToDevice, st));
	CU(cudaStreamSynchronize(st));
	e.dev.cam = dev_camera(cams[0]);
	if ((rc = e.apply())) return rc;
	s->view_count = count;
	s->view_cap = cap;
	return CRGPU_OK;
}

/* ---- render settings between renders ---------------------------------------------------------------------------------------------
 * The kernels read image size, sample count and bounce limit from the descriptor, so publishing it is all they need.  What is sized
 * from the image is swapped here: view 0's framebuffer and the views block (at the view count, cameras and framebuffers), both new and
 * zeroed; the sRGB8 staging buffers go back to the cache and are allocated again at the new size when next used. */
extern "C" int crgpu_scene_set_render(crgpu_scene *s, uint32_t width, uint32_t height, uint32_t sample_count, uint32_t bounces,
                                      const struct crs_camera *cams, uint32_t count) {
	if (!s) return fail(CRGPU_ERR_BAD_ARGUMENT, "scene is NULL");
	if (width == 0 || height == 0 || sample_count == 0) return fail(CRGPU_ERR_BAD_ARGUMENT, "empty image or zero samples");
	if (count != s->view_count) return fail(CRGPU_ERR_BAD_ARGUMENT, "%u cameras for a list of %u views", count, s->view_count);
	const bool resize = width != s->dev.image_width || height != s->dev.image_height;
	if (!cams && resize) return fail(CRGPU_ERR_BAD_ARGUMENT, "a new image size needs a camera for each view");
	for (uint32_t i = 0; cams && i < count; ++i)
		if (cams[i].width != (int32_t)width || cams[i].height != (int32_t)height)
			return fail(CRGPU_ERR_BAD_ARGUMENT, "camera %u is %dx%d, the settings render %ux%u", i, cams[i].width, cams[i].height, width, height);
	if ((uint64_t)width * height > SIZE_MAX / (3u * sizeof(float)) / count)
		return fail(CRGPU_ERR_NOMEM, "%u framebuffers of %ux%u do not fit the address space", count, width, height);
	int rc = drain(s);
	if (rc) return rc;
	const size_t fb_floats = resize ? (size_t)width * height * 3u : s->fb_floats;
	const uint32_t cap = resize ? count : s->view_cap;
	Edit e(s);
	if (resize) {                                      /* new zeroed framebuffers (no views block for one view); the sRGB8 staging goes */
		DevBlock &fb = e.stage(s->fb), &views = e.stage(s->views);
		e.stage(s->fb8);
		e.stage(s->snap8);
		e.stage(s->adapt);                             /* the pixel records are of the old size: a round needs a new reset */
		if ((rc = fb.alloc(s->device, fb_floats * sizeof(float)))) return rc;
		if (count > 1u && (rc = views.alloc(s->device, views_bytes(cap, fb_floats)))) return rc;
		CU(cudaMemsetAsync(fb.p, 0, fb.bytes, s->stream));
		if (count > 1u) CU(cudaMemsetAsync(views_fb(views, cap), 0, (size_t)(count - 1u) * fb_floats * sizeof(float), s->stream));
	}
	std::vector<DevCamera> dc(cams ? count - 1u : 0u);
	for (size_t i = 0; i < dc.size(); ++i) dc[i] = dev_camera(cams[i + 1u]);
	if (!dc.empty()) CU(cudaMemcpyAsync(e.next(s->views).p, dc.data(), dc.size() * sizeof(DevCamera), cudaMemcpyHostToDevice, s->stream));
	CU(cudaStreamSynchronize(s->stream));
	e.dev.image_width = width; e.dev.image_height = height;
	e.dev.sample_count = sample_count; e.dev.bounces = bounces;
	if (cams) e.dev.cam = dev_camera(cams[0]);
	if ((rc = e.apply())) return rc;
	if (resize) {
		s->fb_floats = fb_floats;
		s->view_cap = cap;
		unsigned staged = 2u;                          /* an image staged at the old size is dropped; a pending request stays */
		if (s->stop_host) __atomic_compare_exchange_n(&s->stop_host[3], &staged, 0u, false, __ATOMIC_ACQ_REL, __ATOMIC_ACQUIRE);
	}
	return CRGPU_OK;
}

extern "C" int crgpu_scene_view_count(crgpu_scene *s, uint32_t *count) {
	if (!s || !count) return fail(CRGPU_ERR_BAD_ARGUMENT, "NULL argument");
	*count = s->view_count;
	return CRGPU_OK;
}

extern "C" int crgpu_render_views(crgpu_scene *s, uint32_t first_view, uint32_t view_count, const int *rects, int nrects, int pass_begin,
                                  int pass_count, unsigned flags, struct crgpu_stats *stats) {
	if (!s) return fail(CRGPU_ERR_BAD_ARGUMENT, "scene is NULL");
	if (view_count < 1 || first_view >= s->view_count || view_count > s->view_count - first_view)
		return fail(CRGPU_ERR_BAD_ARGUMENT, "views [%u,%llu) outside the list of %u", first_view, (unsigned long long)first_view + view_count, s->view_count);
	uint64_t npix = 0;
	int rc = tile_set(s, rects, nrects, view_count, &npix);
	if (rc) return rc;
	ViewDesc vd;
	vd.cam0 = &s->dev_copy->cam;
	vd.cams = static_cast<const DevCamera *>(s->views.p);
	vd.fb = views_fb(s->views, s->view_cap);
	vd.fb_floats = s->fb_floats;
	vd.npix = (unsigned)npix;
	vd.view0 = first_view;
	vd.p0 = 0u;
	TileDesc td;
	memset(&td, 0, sizeof td);
	td.pixels = s->pixels.as<uint32_t>();
	return render_call(s, td, npix * view_count, pass_begin, pass_count, flags, stats, &vd);
}

/* ---- adaptive rounds ----------------------------------------------------------------------------------------------------------------
 * The adaptive block: W*H pixel records (AdaptPix, framebuffer order), then the select's scratch for a tile set of up to W*H pixels: the
 * active list, the flags and their inclusive scan, the scan's block sums, and the min / max words. */
struct AdaptParts {
	AdaptPix *recs;
	uint32_t *active;
	unsigned long long *flags, *incl, *sums, *sums2;
	unsigned *mm;
};
static size_t adapt_carve(void *base, size_t npix, AdaptParts *p) {
	size_t off = 0;
	auto take = [&](size_t bytes) { void *q = base ? static_cast<uint8_t *>(base) + off : nullptr; off += align256(bytes); return q; };
	p->recs = (AdaptPix *)take(npix * sizeof(AdaptPix));
	p->active = (uint32_t *)take(npix * 4u);
	p->flags = (unsigned long long *)take(npix * 8u);
	p->incl = (unsigned long long *)take(npix * 8u);
	p->sums = (unsigned long long *)take(8u * (npix / 1024u + 1u));
	p->sums2 = (unsigned long long *)take(8u * (npix / (1024u * 1024u) + 1u));
	p->mm = (unsigned *)take(8u);
	return off;
}

extern "C" int crgpu_adaptive_reset(crgpu_scene *s) {
	if (!s) return fail(CRGPU_ERR_BAD_ARGUMENT, "scene is NULL");
	int rc = drain(s);                                                /* an asynchronous round may still update the records */
	if (rc) return rc;
	const size_t npix = (size_t)s->dev.image_width * s->dev.image_height;
	if (npix > (1ull << 30)) return fail(CRGPU_ERR_UNSUPPORTED, "adaptive rounds need images of at most 2^30 pixels");
	if (!s->adapt_host) {
		void *p = nullptr;
		CU(cudaHostAlloc(&p, 64, cudaHostAllocMapped | cudaHostAllocPortable));
		s->adapt_host = static_cast<unsigned *>(p);
	}
	AdaptParts p;
	if (!s->adapt.p && (rc = s->adapt.alloc(s->device, adapt_carve(nullptr, npix, &p)))) return rc;
	adapt_carve(s->adapt.p, npix, &p);
	crg_launch_adapt_reset(p.recs, npix, s->stream);
	CU(cudaGetLastError());
	CU(cudaStreamSynchronize(s->stream));
	return CRGPU_OK;
}

/* no pixel of the tile set listed twice: K5 would add two passes to it at once.  The last set found clean is remembered. */
static int check_disjoint(crgpu_scene *s, const int *rects, int nrects) {
	std::vector<int> key(rects, rects + 4 * (size_t)nrects);
	if (key == s->adapt_key) return CRGPU_OK;
	const size_t W = s->dev.image_width;
	std::vector<uint8_t> seen(W * s->dev.image_height, 0u);
	for (int i = 0; i < nrects; ++i) {
		const int *r = rects + 4 * i;
		for (int y = r[1]; y < r[3]; ++y)
			for (int x = r[0]; x < r[2]; ++x) {
				uint8_t &b = seen[(size_t)y * W + (size_t)x];
				if (b) return fail(CRGPU_ERR_BAD_ARGUMENT, "tile %d [%d,%d)x[%d,%d) overlaps an earlier tile at (%d, %d)", i, r[0], r[2], r[1], r[3], x, y);
				b = 1u;
			}
	}
	s->adapt_key.swap(key);
	return CRGPU_OK;
}

/* A round's select step over the tile set: test and flag (k_adapt_select), scan, compact (k_adapt_compact), then the one synchronisation.
 * On success p holds the carved adaptive block, whose active list has *count pixels, all at *lo = *hi passes (with none active, *lo =
 * 0xffffffff and *hi = 0).  Refused: fields of a out of range, no adaptive block, a bad or overlapping tile set, and active pixels of
 * different counts (which the compaction leaves unrecorded). */
static int adapt_select(crgpu_scene *s, const int *rects, int nrects, const struct crgpu_adaptive *a, AdaptParts &p, unsigned *count,
                        unsigned *lo, unsigned *hi) {
	if (a->min_passes < 2u || a->round_passes < 1u || a->pass_end < 1u || a->pass_end > s->dev.sample_count)
		return fail(CRGPU_ERR_BAD_ARGUMENT, "min_passes %u (>= 2), round_passes %u (>= 1) or pass_end %u (1 .. %u) out of range", a->min_passes,
		            a->round_passes, a->pass_end, s->dev.sample_count);
	if (!std::isfinite(a->threshold) || a->threshold < 0.f || !std::isfinite(a->floor) || !(a->floor > 0.f))
		return fail(CRGPU_ERR_BAD_ARGUMENT, "threshold %g must be finite and >= 0, floor %g finite and > 0", (double)a->threshold, (double)a->floor);
	if (!s->adapt.p) return fail(CRGPU_ERR_BAD_ARGUMENT, "no adaptive state at this image size: call crgpu_adaptive_reset");
	uint64_t npix = 0;
	int rc = tile_set(s, rects, nrects, 0, &npix);
	if (rc) return rc;
	if ((rc = check_disjoint(s, rects, nrects))) return rc;
	adapt_carve(s->adapt.p, (size_t)s->dev.image_width * s->dev.image_height, &p);
	const AdaptParams ap = { a->min_passes, a->round_passes, a->pass_end, a->threshold, a->floor };
	const int W = (int)s->dev.image_width, H = (int)s->dev.image_height;
	const unsigned n = (unsigned)npix;
	const uint32_t *pixels = s->pixels.as<uint32_t>();
	CU(cudaMemsetAsync(p.mm, 0, 8u, s->stream));
	crg_launch_adapt_select(pixels, n, p.recs, W, H, ap, p.flags, p.mm, s->stream);
	const int scans = crg_scan64(p.flags, p.incl, p.sums, p.sums2, n, s->stream);
	crg_launch_adapt_compact(pixels, n, p.recs, W, H, ap, p.flags, p.incl, p.active, p.mm, s->adapt_host, s->stream);
	CU(cudaGetLastError());
	s->pend_launches += 2u + (uint64_t)scans;
	CU(cudaStreamSynchronize(s->stream));                            /* the round's one synchronisation: the active count and its passes */
	*count = __atomic_load_n(&s->adapt_host[0], __ATOMIC_ACQUIRE);
	*lo = __atomic_load_n(&s->adapt_host[1], __ATOMIC_ACQUIRE);
	*hi = __atomic_load_n(&s->adapt_host[2], __ATOMIC_ACQUIRE);
	if (*count && *lo != *hi)
		return fail(CRGPU_ERR_BAD_ARGUMENT, "the tile set's active pixels hold %u to %u passes: finish the overlapping tile set first", *lo, *hi);
	return CRGPU_OK;
}

extern "C" int crgpu_adaptive_round(crgpu_scene *s, const int *rects, int nrects, const struct crgpu_adaptive *a, unsigned flags,
                                    struct crgpu_stats *stats, uint32_t *active, int *pass_begin, int *pass_end_of_round) {
	if (!s || !a || !active || !pass_begin || !pass_end_of_round) return fail(CRGPU_ERR_BAD_ARGUMENT, "NULL argument");
	AdaptParts p;
	unsigned count = 0u, lo = 0u, hi = 0u;
	int rc = adapt_select(s, rects, nrects, a, p, &count, &lo, &hi);
	if (rc) return rc;
	*active = count;
	if (!count) {
		*pass_begin = *pass_end_of_round = (int)a->pass_end;
		return flags & CRGPU_FLAG_ASYNC ? CRGPU_OK : crgpu_get_stats(s, stats);
	}
	unsigned next = lo < a->min_passes ? a->min_passes : a->min_passes + ((lo - a->min_passes) / a->round_passes + 1u) * a->round_passes;
	if (next > a->pass_end) next = a->pass_end;
	*pass_begin = (int)lo;
	*pass_end_of_round = (int)next;
	TileDesc td;
	memset(&td, 0, sizeof td);
	td.pixels = p.active;
	return render_call(s, td, count, (int)lo, (int)(next - lo), flags, stats, nullptr, p.recs);
}

extern "C" int crgpu_adaptive_read(crgpu_scene *s, uint32_t *passes, float *err) {
	if (!s) return fail(CRGPU_ERR_BAD_ARGUMENT, "scene is NULL");
	if (!s->adapt.p) return fail(CRGPU_ERR_BAD_ARGUMENT, "no adaptive state at this image size: call crgpu_adaptive_reset");
	const size_t npix = (size_t)s->dev.image_width * s->dev.image_height;
	std::vector<AdaptPix> h(npix);
	CU(cudaSetDevice(s->device));
	CU(cudaMemcpyAsync(h.data(), s->adapt.p, npix * sizeof(AdaptPix), cudaMemcpyDeviceToHost, s->stream));
	CU(cudaStreamSynchronize(s->stream));
	for (size_t i = 0; i < npix; ++i) {
		if (passes) passes[i] = h[i].n & ~CRG_ADAPT_DONE;
		if (err) err[i] = h[i].err;
	}
	return CRGPU_OK;
}

/* ---- test entry points of K5 and of a round's select (include/crgpu.h) ---------------------------------------------------------- */
static_assert(sizeof(crgpu_adaptive_record) == sizeof(AdaptPix) && CRGPU_ADAPTIVE_DONE == CRG_ADAPT_DONE, "crgpu_adaptive_record is AdaptPix");

extern "C" int crgpu_accumulate_samples(crgpu_scene *s, const int *rects, int nrects, int pass_begin, int pass_count, int order, int adaptive,
                                        const float *L, uint32_t *pixels_out) {
	if (!s || !L) return fail(CRGPU_ERR_BAD_ARGUMENT, "NULL argument");
	if (order < -1 || order >= CRG_PATH_ORDERS) return fail(CRGPU_ERR_BAD_ARGUMENT, "path order %d outside -1 .. %d", order, CRG_PATH_ORDERS - 1);
	if (adaptive && !s->adapt.p) return fail(CRGPU_ERR_BAD_ARGUMENT, "no adaptive state at this image size: call crgpu_adaptive_reset");
	if (pass_begin < 0 || pass_count < 0 || (uint64_t)pass_begin + (uint64_t)pass_count > s->dev.sample_count)
		return fail(CRGPU_ERR_BAD_ARGUMENT, "passes [%d,%d) outside [0,%u)", pass_begin, pass_begin + pass_count, s->dev.sample_count);
	uint64_t npix = 0;
	int rc = tile_set(s, rects, nrects, 0, &npix);
	if (rc) return rc;
	const uint64_t paths = npix * (uint64_t)pass_count;
	if (paths > s->max_paths)
		return fail(CRGPU_ERR_BAD_ARGUMENT, "%llu pixels x %d passes are more than the %llu paths in flight", (unsigned long long)npix, pass_count,
		            (unsigned long long)s->max_paths);
	if ((rc = drain(s)) || (rc = alloc_wave(s, paths ? paths : 1, 1))) return rc;
	const PathOrder po = order < 0 ? crg_path_order() : crg_path_order_of(order);
	std::vector<float4> h(paths);
	for (uint64_t px = 0; px < npix; ++px)
		for (int pl = 0; pl < pass_count; ++pl) {
			const float *v = L + (px * (uint64_t)pass_count + (uint64_t)pl) * 4u;
			h[crg_path_id((unsigned)pl, (unsigned)px, (unsigned)npix, (unsigned)pass_count, po.p, po.q)] = make_float4(v[0], v[1], v[2], v[3]);
		}
	if (paths) {
		CU(cudaMemcpyAsync(s->wb.L, h.data(), paths * sizeof(float4), cudaMemcpyHostToDevice, s->stream));
		TileDesc td;
		memset(&td, 0, sizeof td);
		td.pixels = s->pixels.as<uint32_t>();
		td.npix = (unsigned)npix;
		td.order = po;
		td.pass_begin = pass_begin;
		td.pass_count = pass_count;
		AdaptParts p = {};
		if (adaptive) adapt_carve(s->adapt.p, (size_t)s->dev.image_width * s->dev.image_height, &p);
		crg_launch_accumulate(s->fb.as<float>(), s->wb.L, td, (int)s->dev.image_width, (int)s->dev.image_height, s->sm_count * 8, s->stream, nullptr, 0,
		                      nullptr, nullptr, p.recs);
		CU(cudaGetLastError());
		s->pend_launches += 1u;
	}
	if (pixels_out && npix) CU(cudaMemcpyAsync(pixels_out, s->pixels.p, npix * sizeof(uint32_t), cudaMemcpyDeviceToHost, s->stream));
	CU(cudaStreamSynchronize(s->stream));
	return CRGPU_OK;
}

extern "C" int crgpu_adaptive_write(crgpu_scene *s, const struct crgpu_adaptive_record *recs) {
	if (!s || !recs) return fail(CRGPU_ERR_BAD_ARGUMENT, "NULL argument");
	if (!s->adapt.p) return fail(CRGPU_ERR_BAD_ARGUMENT, "no adaptive state at this image size: call crgpu_adaptive_reset");
	int rc = drain(s);
	if (rc) return rc;
	const size_t npix = (size_t)s->dev.image_width * s->dev.image_height;
	CU(cudaMemcpyAsync(s->adapt.p, recs, npix * sizeof(AdaptPix), cudaMemcpyHostToDevice, s->stream));
	CU(cudaStreamSynchronize(s->stream));
	return CRGPU_OK;
}

extern "C" int crgpu_adaptive_records(crgpu_scene *s, struct crgpu_adaptive_record *recs_out) {
	if (!s || !recs_out) return fail(CRGPU_ERR_BAD_ARGUMENT, "NULL argument");
	if (!s->adapt.p) return fail(CRGPU_ERR_BAD_ARGUMENT, "no adaptive state at this image size: call crgpu_adaptive_reset");
	int rc = drain(s);
	if (rc) return rc;
	const size_t npix = (size_t)s->dev.image_width * s->dev.image_height;
	CU(cudaMemcpyAsync(recs_out, s->adapt.p, npix * sizeof(AdaptPix), cudaMemcpyDeviceToHost, s->stream));
	CU(cudaStreamSynchronize(s->stream));
	return CRGPU_OK;
}

extern "C" int crgpu_adaptive_select(crgpu_scene *s, const int *rects, int nrects, const struct crgpu_adaptive *a, uint32_t *active_out,
                                     uint32_t *count_out, uint32_t *lo_out, uint32_t *hi_out) {
	if (!s || !a || !active_out || !count_out || !lo_out || !hi_out) return fail(CRGPU_ERR_BAD_ARGUMENT, "NULL argument");
	AdaptParts p;
	unsigned count = 0u, lo = 0u, hi = 0u;
	int rc = adapt_select(s, rects, nrects, a, p, &count, &lo, &hi);
	if (rc) return rc;
	if (count) {
		CU(cudaMemcpyAsync(active_out, p.active, (size_t)count * sizeof(uint32_t), cudaMemcpyDeviceToHost, s->stream));
		CU(cudaStreamSynchronize(s->stream));
	}
	*count_out = count; *lo_out = lo; *hi_out = hi;
	return CRGPU_OK;
}

static int check_view(const crgpu_scene *s, uint32_t view) {
	if (!s) return fail(CRGPU_ERR_BAD_ARGUMENT, "scene is NULL");
	if (view >= s->view_count) return fail(CRGPU_ERR_BAD_ARGUMENT, "view %u outside the list of %u", view, s->view_count);
	return CRGPU_OK;
}

extern "C" int crgpu_view_clear(crgpu_scene *s, uint32_t view) {
	int rc = check_view(s, view);
	if (rc) return rc;
	CU(cudaSetDevice(s->device));
	CU(cudaMemsetAsync(view_fb(s, view), 0, s->fb_floats * sizeof(float), s->stream));
	CU(cudaStreamSynchronize(s->stream));
	return CRGPU_OK;
}

extern "C" int crgpu_view_read(crgpu_scene *s, uint32_t view, float *host_rgb) {
	int rc = check_view(s, view);
	if (rc) return rc;
	if (!host_rgb) return fail(CRGPU_ERR_BAD_ARGUMENT, "NULL argument");
	CU(cudaSetDevice(s->device));
	CU(cudaMemcpyAsync(host_rgb, view_fb(s, view), s->fb_floats * sizeof(float), cudaMemcpyDeviceToHost, s->stream));
	CU(cudaStreamSynchronize(s->stream));
	return CRGPU_OK;
}

/* view v's image as sRGB8 (view 0: the scene's framebuffer), through fb8 */
static int to_srgb8(crgpu_scene *s, uint32_t v, uint8_t *host_rgb8) {
	CU(cudaSetDevice(s->device));
	int rc = alloc_srgb8(s, s->fb8);
	if (rc) return rc;
	crg_launch_to_srgb8(view_fb(s, v), s->fb8.as<uint8_t>(), s->fb_floats, s->sm_count * 8, s->stream);
	CU(cudaGetLastError());
	CU(cudaMemcpyAsync(host_rgb8, s->fb8.p, s->fb_floats, cudaMemcpyDeviceToHost, s->stream));
	CU(cudaStreamSynchronize(s->stream));
	return CRGPU_OK;
}

extern "C" int crgpu_view_to_srgb8(crgpu_scene *s, uint32_t view, uint8_t *host_rgb8) {
	int rc = check_view(s, view);
	if (rc) return rc;
	if (!host_rgb8) return fail(CRGPU_ERR_BAD_ARGUMENT, "NULL argument");
	return to_srgb8(s, view, host_rgb8);
}

extern "C" int crgpu_get_stats(crgpu_scene *s, struct crgpu_stats *stats) {
	if (!s) return fail(CRGPU_ERR_BAD_ARGUMENT, "scene is NULL");
	CU(cudaSetDevice(s->device));
	unsigned long long h[8];
	CU(cudaMemcpyAsync(h, s->wb.stats, sizeof h, cudaMemcpyDeviceToHost, s->stream));
	CU(cudaStreamSynchronize(s->stream));
	if (h[7] != s->fetched[7]) {
		memcpy(s->fetched, h, sizeof h);
		return fail(CRGPU_ERR_CUDA, "traversal watchdog: %llu ray(s) exceeded the step limit (corrupt BVH?)", h[7]);
	}
	if (stats) {
		memset(stats, 0, sizeof *stats);
		stats->paths = s->pend_paths + (h[5] - s->fetched[5]);   /* + the passes armed calls committed */
		stats->rays = h[0] - s->fetched[0]; stats->node_pairs = h[1] - s->fetched[1]; stats->tri_tests = h[2] - s->fetched[2];
		stats->sphere_tests = h[3] - s->fetched[3]; stats->inst_visits = h[4] - s->fetched[4];
		stats->kernel_launches = s->pend_launches;
		stats->trace_ms = s->pend_trace_ms; stats->shade_ms = s->pend_shade_ms; stats->total_ms = s->pend_total_ms;
	}
	memcpy(s->fetched, h, sizeof h);
	s->pend_paths = s->pend_launches = 0; s->pend_trace_ms = s->pend_shade_ms = s->pend_total_ms = 0.f;
	return CRGPU_OK;
}

extern "C" int crgpu_set_stream(crgpu_scene *s, void *cuda_stream) {
	if (!s) return fail(CRGPU_ERR_BAD_ARGUMENT, "scene is NULL");
	CU(cudaSetDevice(s->device));
	CU(cudaStreamSynchronize(s->stream));
	s->stream = static_cast<cudaStream_t>(cuda_stream);      /* NULL is a valid handle: the legacy default stream */
	return CRGPU_OK;
}

extern "C" int crgpu_use_own_stream(crgpu_scene *s) {
	if (!s) return fail(CRGPU_ERR_BAD_ARGUMENT, "scene is NULL");
	CU(cudaSetDevice(s->device));
	CU(cudaStreamSynchronize(s->stream));
	s->stream = s->own_stream;
	return CRGPU_OK;
}

extern "C" int crgpu_framebuffer_clear(crgpu_scene *s) {
	if (!s) return fail(CRGPU_ERR_BAD_ARGUMENT, "scene is NULL");
	CU(cudaSetDevice(s->device));
	CU(cudaMemsetAsync(s->fb.p, 0, s->fb.bytes, s->stream));
	CU(cudaStreamSynchronize(s->stream));
	return CRGPU_OK;
}

static int fb_copy(crgpu_scene *s, float *host, int x0, int y0, int x1, int y1, bool to_host) {
	if (!s || !host) return fail(CRGPU_ERR_BAD_ARGUMENT, "NULL argument");
	CU(cudaSetDevice(s->device));
	const size_t W = s->dev.image_width, H = s->dev.image_height;
	if (x1 <= x0) { x0 = 0; y0 = 0; x1 = (int)W; y1 = (int)H; }
	int rc = check_rect(s, x0, y0, x1, y1);
	if (rc) return rc;
	/* rows y0..y1-1 (y up) are storage rows H-y1 .. H-1-y0 */
	const size_t row0 = H - (size_t)y1, rows = (size_t)(y1 - y0);
	const size_t off = (row0 * W + (size_t)x0) * 3u;
	const size_t pitch = W * 3u * sizeof(float), width = (size_t)(x1 - x0) * 3u * sizeof(float);
	if (to_host) CU(cudaMemcpy2DAsync(host + off, pitch, s->fb.as<float>() + off, pitch, width, rows, cudaMemcpyDeviceToHost, s->stream));
	else CU(cudaMemcpy2DAsync(s->fb.as<float>() + off, pitch, host + off, pitch, width, rows, cudaMemcpyHostToDevice, s->stream));
	CU(cudaStreamSynchronize(s->stream));
	return CRGPU_OK;
}
extern "C" int crgpu_framebuffer_read(crgpu_scene *s, float *host_rgb, int x0, int y0, int x1, int y1) {
	return fb_copy(s, host_rgb, x0, y0, x1, y1, true);
}
extern "C" int crgpu_framebuffer_write(crgpu_scene *s, const float *host_rgb, int x0, int y0, int x1, int y1) {
	return fb_copy(s, const_cast<float *>(host_rgb), x0, y0, x1, y1, false);
}

extern "C" int crgpu_framebuffer_to_srgb8(crgpu_scene *s, uint8_t *host_rgb8) {
	if (!s || !host_rgb8) return fail(CRGPU_ERR_BAD_ARGUMENT, "NULL argument");
	return to_srgb8(s, 0, host_rgb8);
}

extern "C" int crgpu_framebuffer_device_ptr(crgpu_scene *s, void **dev_ptr, size_t *bytes) {
	if (!s || !dev_ptr) return fail(CRGPU_ERR_BAD_ARGUMENT, "NULL argument");
	*dev_ptr = s->fb.p;
	if (bytes) *bytes = s->fb_floats * sizeof(float);
	return CRGPU_OK;
}

extern "C" int crgpu_scene_info(crgpu_scene *s, int *device, int *width, int *height) {
	if (!s) return fail(CRGPU_ERR_BAD_ARGUMENT, "scene is NULL");
	if (device) *device = s->device;
	if (width) *width = (int)s->dev.image_width;
	if (height) *height = (int)s->dev.image_height;
	return CRGPU_OK;
}

/* ---- test entries: a batch of rays or path states in half 0 of wave set 0 -----------------------------------------------------------
 * stage_half0 takes the counters of earlier work (so that the stats afterwards are this batch's), makes room for n paths, loads stA,
 * stB and (path states) stC, sets the live count to n and clears K2's histogram.  read_trace_records copies K2's write-back of the
 * batch (crg_launch_trace_records) to the host and waits for the stream. */
static int stage_half0(crgpu_scene *s, uint32_t n, const float4 *a, const float4 *b, const uint4 *c) {
	int rc = crgpu_get_stats(s, nullptr);
	if (rc) return rc;
	rc = alloc_wave(s, n ? n : 1, 1);
	if (rc) return rc;
	const WaveBuffers &wb = s->wb;
	cudaStream_t st = s->stream;
	const unsigned counts[5] = { n, 0u, 0u, 0u, 0u };
	CU(cudaMemcpyAsync(wb.stA[0], a, (size_t)n * sizeof(float4), cudaMemcpyHostToDevice, st));
	CU(cudaMemcpyAsync(wb.stB[0], b, (size_t)n * sizeof(float4), cudaMemcpyHostToDevice, st));
	if (c) CU(cudaMemcpyAsync(wb.stC[0], c, (size_t)n * sizeof(uint4), cudaMemcpyHostToDevice, st));
	CU(cudaMemcpyAsync(wb.counts, counts, sizeof counts, cudaMemcpyHostToDevice, st));
	CU(cudaMemsetAsync(wb.hist, 0, 1024 * sizeof(unsigned), st));
	return CRGPU_OK;
}
static int read_trace_records(crgpu_scene *s, uint32_t n, struct crgpu_ray_record *out, const char *entry) {
	if (!n) return CRGPU_OK;
	void *drec = nullptr;
	CU(cudaMalloc(&drec, (size_t)n * sizeof *out));
	crg_launch_trace_records(s->dev, s->wb, n, drec, s->sm_count * 8, s->stream);
	cudaError_t e = cudaGetLastError();
	if (e == cudaSuccess) e = cudaMemcpyAsync(out, drec, (size_t)n * sizeof *out, cudaMemcpyDeviceToHost, s->stream);
	if (e == cudaSuccess) e = cudaStreamSynchronize(s->stream);
	cudaFree(drec);
	if (e != cudaSuccess) return fail(CRGPU_ERR_CUDA, "%s: %s", entry, cudaGetErrorString(e));
	return CRGPU_OK;
}

/* Closest hits of a ray batch through the production K2 (k_trace, by the launch path and launch shape of a frame) and K4. */
extern "C" int crgpu_trace_rays(crgpu_scene *s, const float *rays, uint32_t n, const struct crgpu_trace_opts *opts,
								struct crgpu_ray_record *records_out, uint32_t *perm_out, uint32_t *misses_out, struct crgpu_stats *stats_out) {
	if (!s || !opts || (n && (!rays || !records_out || !perm_out)) || n > (1u << 30)) return fail(CRGPU_ERR_BAD_ARGUMENT, "bad argument");
	TraceKnobs kn;
	kn.minb = opts->minb; kn.defer = opts->defer; kn.refill = opts->refill; kn.burst = opts->burst; kn.inst_min = opts->inst_min;
	if (kn.minb < 2 || kn.minb > 4 || kn.defer < 0 || kn.defer > 2 || kn.refill < 1 || kn.refill > 32 || kn.burst < 1 || kn.inst_min < 1 || kn.inst_min > 32)
		return fail(CRGPU_ERR_BAD_ARGUMENT, "trace options out of range");
	if (opts->order) {                                  /* K2 reads rays through the order: it must be a permutation of [0, n) */
		std::vector<uint8_t> seen(n, 0);
		for (uint32_t i = 0; i < n; ++i) {
			if (opts->order[i] >= n || seen[opts->order[i]]) return fail(CRGPU_ERR_BAD_ARGUMENT, "order is not a permutation of [0, %u)", n);
			seen[opts->order[i]] = 1;
		}
	}
	CU(cudaSetDevice(s->device));
	std::vector<float4> a(n), b(n);
	for (uint32_t i = 0; i < n; ++i) {
		const float *r = rays + 6 * (size_t)i;
		a[i] = make_float4(r[0], r[1], r[2], r[3]);
		b[i] = make_float4(r[4], r[5], 1.0f, 1.0f);
	}
	int rc = stage_half0(s, n, a.data(), b.data(), nullptr);
	if (rc) return rc;
	const WaveBuffers &wb = s->wb;
	cudaStream_t st = s->stream;
	if (opts->order) CU(cudaMemcpyAsync(wb.perm2, opts->order, (size_t)n * sizeof(uint32_t), cudaMemcpyHostToDevice, st));
	/* poison: no write-back produces a negative distance or the instance index -1515870811, and K4 must overwrite all of perm.
	 * Every 8-bit value is some ray's key, so a key left behind shows only as a key that differs from the expected one; the
	 * write-back stores hit, instance and key together, so a ray it missed also keeps the hit and instance poison */
	CU(cudaMemsetAsync(wb.hit, 0xA5, (size_t)n * sizeof(float4), st));
	CU(cudaMemsetAsync(wb.hitInst, 0xA5, (size_t)n * sizeof(int), st));
	CU(cudaMemsetAsync(wb.hitKey, 0xA5, (size_t)n, st));
	CU(cudaMemsetAsync(wb.perm, 0xFF, (size_t)n * sizeof(unsigned), st));
	crg_launch_trace(s->dev, wb, 0, opts->count != 0, opts->order != nullptr, kn, st);
	crg_launch_bucket(wb, 0, s->sm_count * 8, nullptr, 0, st);      /* buckets in key order */
	CU(cudaGetLastError());
	rc = read_trace_records(s, n, records_out, "trace_rays");
	if (rc) return rc;
	unsigned cnt[5];
	cudaError_t e = cudaSuccess;
	if (n) e = cudaMemcpyAsync(perm_out, wb.perm, (size_t)n * sizeof(uint32_t), cudaMemcpyDeviceToHost, st);
	if (e == cudaSuccess) e = cudaMemcpyAsync(cnt, wb.counts, sizeof cnt, cudaMemcpyDeviceToHost, st);
	if (e == cudaSuccess) e = cudaStreamSynchronize(st);
	if (e != cudaSuccess) return fail(CRGPU_ERR_CUDA, "trace_rays: %s", cudaGetErrorString(e));
	if (misses_out) *misses_out = cnt[4];
	return crgpu_get_stats(s, stats_out);               /* fails if the traversal watchdog fired */
}

extern "C" int crgpu_trace_kat(crgpu_scene *s, const int32_t *xyp, int count, void *records_out) {
	if (!s || !xyp || !records_out || count < 0) return fail(CRGPU_ERR_BAD_ARGUMENT, "bad argument");
	if (count == 0) return CRGPU_OK;
	CU(cudaSetDevice(s->device));
	int32_t *dx = nullptr;
	void *dk = nullptr;
	CU(cudaMalloc((void **)&dx, (size_t)count * 3 * sizeof(int32_t)));
	CU(cudaMalloc((void **)&dk, (size_t)count * CRG_HITKAT_BYTES));
	CU(cudaMemcpyAsync(dx, xyp, (size_t)count * 3 * sizeof(int32_t), cudaMemcpyHostToDevice, s->stream));
	crg_launch_kat(s->dev_copy, dx, count, dk, s->stream);
	cudaError_t e = cudaGetLastError();
	if (e == cudaSuccess) e = cudaMemcpyAsync(records_out, dk, (size_t)count * CRG_HITKAT_BYTES, cudaMemcpyDeviceToHost, s->stream);
	if (e == cudaSuccess) e = cudaStreamSynchronize(s->stream);
	cudaFree(dx); cudaFree(dk);
	if (e != cudaSuccess) return fail(CRGPU_ERR_CUDA, "trace_kat: %s", cudaGetErrorString(e));
	return CRGPU_OK;
}

/* One bounce of a batch of path states through the frame's own bounce sequence (enqueue_bounce): K2 -> K4 -> K3 (and K4b when a
 * sort mode is set and another bounce follows), or the tail kernel.  The states go into the current half
 * of the wave buffers with id = their index (| CRG_ID_HAS_L where has_l is set) and L as given; the other half is poisoned.  Each
 * result is found by the id K3 compacted it with. */
#define CRG_ID_HAS_L_HOST 0x80000000u
extern "C" int crgpu_shade_rays(crgpu_scene *s, const struct crgpu_path_state *states, uint32_t n, const struct crgpu_shade_opts *opts,
								struct crgpu_shade_result *results, uint32_t *perm2_out, uint32_t *survivors_out, uint32_t *box_out) {
	if (!s || !opts || (n && (!states || !results || !perm2_out)) || !survivors_out || n > (1u << 30)) return fail(CRGPU_ERR_BAD_ARGUMENT, "bad argument");
	ShadeKnobs kn;
	kn.minb = opts->minb; kn.split = opts->split; kn.prefetch = opts->prefetch;
	kn.generic_only = opts->generic_only; kn.flat_minb = opts->minb;      /* both hit kernels at the bound the caller names */
	if (kn.minb < 2 || kn.minb > 4 || kn.split < 0 || kn.split > 1 || kn.prefetch < 0 || kn.prefetch > 1 || opts->dirmode < 0 || opts->dirmode > 4 ||
		kn.generic_only < 0 || kn.generic_only > 1 ||
		opts->depth < 0 || opts->max_depth < 1 || opts->depth >= opts->max_depth)
		return fail(CRGPU_ERR_BAD_ARGUMENT, "shade options out of range");
	CU(cudaSetDevice(s->device));
	const bool xnodes = s->xnodes || opts->complete_interpreter;
	std::vector<float4> a(n), b(n), L(n);
	std::vector<uint4> c(n);
	for (uint32_t i = 0; i < n; ++i) {
		const crgpu_path_state &p = states[i];
		a[i] = make_float4(p.o[0], p.o[1], p.o[2], p.d[0]);
		b[i] = make_float4(p.d[1], p.d[2], p.weight[0], p.weight[1]);
		uint32_t wb32;
		memcpy(&wb32, &p.weight[2], 4);
		c[i] = make_uint4(wb32, i | (p.has_l ? CRG_ID_HAS_L_HOST : 0u), (uint32_t)(p.rng & 0xffffffffull), (uint32_t)(p.rng >> 32));
		L[i] = make_float4(p.L[0], p.L[1], p.L[2], 0.0f);
	}
	int rc = stage_half0(s, n, a.data(), b.data(), c.data());
	if (rc) return rc;
	const WaveBuffers &wb = s->wb;
	cudaStream_t st = s->stream;
	const size_t n4 = (size_t)n * sizeof(float4);
	if (n) {
		CU(cudaMemcpyAsync(wb.L, L.data(), n4, cudaMemcpyHostToDevice, st));
		CU(cudaMemsetAsync(wb.stA[1], 0xA5, n4, st));
		CU(cudaMemsetAsync(wb.stB[1], 0xA5, n4, st));
		CU(cudaMemsetAsync(wb.stC[1], 0xA5, n4, st));
		CU(cudaMemsetAsync(wb.hit, 0xA5, n4, st));
		CU(cudaMemsetAsync(wb.hitInst, 0xA5, (size_t)n * sizeof(int), st));
		CU(cudaMemsetAsync(wb.dirKey, 0xA5, (size_t)n, st));
		CU(cudaMemsetAsync(wb.perm2, 0xFF, (size_t)n * sizeof(unsigned), st));
	}
	const int depth = opts->depth, maxDepth = opts->max_depth;
	const int box_slot = depth < CRG_BOX_SLOTS ? depth : CRG_BOX_SLOTS - 1;
	unsigned box[12];
	CU(cudaMemcpyAsync(box, wb.box + 12 * box_slot, sizeof box, cudaMemcpyDeviceToHost, st));
	if (opts->tail) crg_launch_tail(s->dev_copy, wb, 0, depth, maxDepth, xnodes, st);
	else enqueue_bounce(s, wb, 0, depth, maxDepth, opts->dirmode, false, false, xnodes, crg_trace_knobs_env(), kn, st, nullptr);
	CU(cudaGetLastError());
	std::vector<crgpu_ray_record> rec(n);
	if (!opts->tail) {
		rc = read_trace_records(s, n, rec.data(), "shade_rays");
		if (rc) return rc;
	}
	std::vector<float4> a2(n), b2(n), L2(n);
	std::vector<uint4> c2(n);
	std::vector<uint8_t> dk(n);
	unsigned cnt[5];
	cudaError_t e = cudaMemcpyAsync(cnt, wb.counts, sizeof cnt, cudaMemcpyDeviceToHost, st);
	if (e == cudaSuccess) e = cudaStreamSynchronize(st);
	const uint32_t surv = opts->tail ? cnt[0] : cnt[1];
	if (e == cudaSuccess && surv > n) return fail(CRGPU_ERR_CUDA, "shade_rays: %u survivors of %u paths", surv, n);
	const int half = opts->tail ? 0 : 1;
	if (e == cudaSuccess && surv) {
		e = cudaMemcpyAsync(a2.data(), half ? wb.stA[1] : wb.stA[0], (size_t)surv * sizeof(float4), cudaMemcpyDeviceToHost, st);
		if (e == cudaSuccess) e = cudaMemcpyAsync(b2.data(), half ? wb.stB[1] : wb.stB[0], (size_t)surv * sizeof(float4), cudaMemcpyDeviceToHost, st);
		if (e == cudaSuccess) e = cudaMemcpyAsync(c2.data(), half ? wb.stC[1] : wb.stC[0], (size_t)surv * sizeof(uint4), cudaMemcpyDeviceToHost, st);
		if (e == cudaSuccess) e = cudaMemcpyAsync(dk.data(), wb.dirKey, surv, cudaMemcpyDeviceToHost, st);
		if (e == cudaSuccess) e = cudaMemcpyAsync(perm2_out, wb.perm2, (size_t)surv * sizeof(uint32_t), cudaMemcpyDeviceToHost, st);
	}
	if (e == cudaSuccess && n) e = cudaMemcpyAsync(L2.data(), wb.L, n4, cudaMemcpyDeviceToHost, st);
	if (e == cudaSuccess) e = cudaStreamSynchronize(st);
	if (e != cudaSuccess) return fail(CRGPU_ERR_CUDA, "shade_rays: %s", cudaGetErrorString(e));
	for (uint32_t i = 0; i < n; ++i) {
		crgpu_shade_result &r = results[i];
		memset(&r, 0, sizeof r);
		if (!opts->tail) r.rec = rec[i];
		else { r.rec.inst = -2; r.rec.poly = -2; }
		r.slot = 0xffffffffu;
		r.dir_key = 0xffffffffu;
		memcpy(r.next.L, &L2[i], 12);
	}
	for (uint32_t k = 0; k < surv; ++k) {
		const uint32_t id = c2[k].y & ~CRG_ID_HAS_L_HOST;
		if (id >= n || results[id].alive) return fail(CRGPU_ERR_CUDA, "shade_rays: survivor %u carries id %u (duplicate or out of range)", k, c2[k].y);
		crgpu_shade_result &r = results[id];
		r.alive = 1;
		r.slot = k;
		r.dir_key = dk[k];
		r.next.o[0] = a2[k].x; r.next.o[1] = a2[k].y; r.next.o[2] = a2[k].z; r.next.d[0] = a2[k].w;
		r.next.d[1] = b2[k].x; r.next.d[2] = b2[k].y; r.next.weight[0] = b2[k].z; r.next.weight[1] = b2[k].w;
		memcpy(&r.next.weight[2], &c2[k].x, 4);
		r.next.has_l = (c2[k].y & CRG_ID_HAS_L_HOST) ? 1u : 0u;
		r.next.rng = (uint64_t)c2[k].z | ((uint64_t)c2[k].w << 32);
	}
	*survivors_out = surv;
	if (box_out) memcpy(box_out, box, sizeof box);
	return crgpu_get_stats(s, nullptr);
}

extern "C" int crgpu_path_order_map(int order, uint32_t npix, uint32_t pass_count, uint32_t *pass_out, uint32_t *pixel_out, uint32_t *id_out,
                                    uint32_t w, uint32_t h, uint32_t *xy_out) {
	if (order < 0 || order >= CRG_PATH_ORDERS || (uint64_t)npix * pass_count > 0xffffffffull || (uint64_t)w * h > 0xffffffffull || w > 65535u || h > 65535u)
		return fail(CRGPU_ERR_BAD_ARGUMENT, "bad argument");
	const PathOrder o = crg_path_order_of(order);
	const uint32_t n = npix * pass_count;
	for (uint32_t id = 0; id < n; ++id) {
		unsigned pl, px;
		crg_path_pass_pixel(id, npix, pass_count, o.p, o.q, pl, px);
		if (pass_out) pass_out[id] = pl;
		if (pixel_out) pixel_out[id] = px;
		if (id_out) id_out[id] = crg_path_id(id / npix, id % npix, npix, pass_count, o.p, o.q);
	}
	const uint32_t m = w * h;
	for (uint32_t i = 0; xy_out && i < m; ++i) {
		unsigned x = i % w, y = i / w;
		if (o.blocked) crg_block_xy(i, w, h, x, y);
		xy_out[i] = x | y << 16;
	}
	return CRGPU_OK;
}

extern "C" int crgpu_libm_eval(int device, int fn, const float *x, const float *y, float *out, uint32_t n) {
	if (fn < 0 || fn >= CRGPU_LIBM_COUNT || (n && (!x || !y || !out))) return fail(CRGPU_ERR_BAD_ARGUMENT, "bad argument");
	if (n == 0) return CRGPU_OK;
	CU(cudaSetDevice(device));
	float *d = nullptr;
	CU(cudaMalloc((void **)&d, (size_t)n * 3 * sizeof(float)));
	cudaError_t e = cudaMemcpy(d, x, (size_t)n * sizeof(float), cudaMemcpyHostToDevice);
	if (e == cudaSuccess) e = cudaMemcpy(d + n, y, (size_t)n * sizeof(float), cudaMemcpyHostToDevice);
	if (e == cudaSuccess) { crg_launch_libm(fn, d, d + n, d + 2 * (size_t)n, n, 0); e = cudaGetLastError(); }
	if (e == cudaSuccess) e = cudaMemcpy(out, d + 2 * (size_t)n, (size_t)n * sizeof(float), cudaMemcpyDeviceToHost);
	cudaFree(d);
	if (e != cudaSuccess) return fail(CRGPU_ERR_CUDA, "libm_eval: %s", cudaGetErrorString(e));
	return CRGPU_OK;
}
