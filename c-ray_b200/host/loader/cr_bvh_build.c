/*
 * cr_bvh_build.c — binned-SAH BVH construction for the scene loader (host side, runs once per scene).
 *
 * The GPU traversal kernels consume exactly the tree the reference builds (node order, leaf ranges and
 * primitive order decide which triangle wins a tie), so this builder follows the algorithm of reference
 * src/accelerators/bvh.c:96-296 decision for decision: 32 bins per axis, right-to-left then left-to-right
 * sweeps, cheapest axis with ties going to the lower axis, leaf cost area*(n - 1.5), approximate-median
 * fallback above 16 primitives, in-place two-pointer partition, children allocated as a pair, depth cap 64.
 * Float expressions keep the reference's association; float->unsigned conversions follow x86-64 cvttss2si.
 * The recursion is replaced by an explicit work stack (same visiting order: left subtree first), and large inputs are
 * built by several threads with a layout pass that restores the serial node numbering.
 */
#include "cr_loader_int.h"
#include "../../../include/crloader.h"
#include <stdlib.h>
#include <string.h>
#include <pthread.h>
#include <unistd.h>

#define MAX_DEPTH      64
#define MAX_LEAF_SIZE  16
#define TRAVERSAL_COST 1.5f
#define BIN_COUNT      32

struct bin { bbox3 bbox; unsigned count; float cost; };

/* (unsigned)f as GCC compiles it on x86-64: cvttss2si to 64 bits, low 32 bits kept; NaN/overflow give 0 */
static inline unsigned f2u(float f) {
	if (!(f > -9.2233720e18f && f < 9.2233720e18f)) return 0u;
	return (unsigned)(long long)f;
}

/* bvh.c:89-95 with `BIN_COUNT / (max - min)` hoisted out of the per-primitive loop (same operands, same quotient) */
static inline unsigned bin_index(float coord, float lo, float centerToBin) {
	float floatIndex = (coord - lo) * centerToBin;
	unsigned b = f2u(floatIndex < 0 ? 0 : floatIndex);
	return b >= BIN_COUNT ? BIN_COUNT - 1 : b;
}

static inline float axis_of(const vec3 *v, int axis) { return axis == 0 ? v->x : (axis == 1 ? v->y : v->z); }

static inline void store_bbox(struct crs_bvh_node *n, const bbox3 *b) {
	n->bounds[0] = b->min.x; n->bounds[1] = b->max.x;
	n->bounds[2] = b->min.y; n->bounds[3] = b->max.y;
	n->bounds[4] = b->min.z; n->bounds[5] = b->max.z;
}

static inline void make_leaf(struct crs_bvh_node *n, unsigned begin, unsigned count) {
	n->first_child_or_prim = begin;
	n->prim_count_leaf = CRS_BVH_LEAF_BIT | (count & CRS_BVH_COUNT_MASK);
}

struct builder { const bbox3 *bboxes; const vec3 *centers; int32_t *prims; };

/* Bin filling (bvh.c:158-171) for prims[begin,end) on the three axes. */
static void fill_bins(const struct builder *B, const float bounds[6], unsigned begin, unsigned end, struct bin bins[3][BIN_COUNT]) {
	for (int axis = 0; axis < 3; ++axis) {
		struct bin *ab = bins[axis];
		for (int i = 0; i < BIN_COUNT; ++i) { ab[i].bbox = crl_empty_bbox; ab[i].count = 0; }
		const float lo = bounds[axis * 2], scale = BIN_COUNT / (bounds[axis * 2 + 1] - lo);
		for (unsigned i = begin; i < end; ++i) {
			const int p = B->prims[i];
			struct bin *b = &ab[bin_index(axis_of(&B->centers[p], axis), lo, scale)];
			bbox_extend(&b->bbox, &B->bboxes[p]);
			b->count++;
		}
	}
}

/* The same for the few huge ranges at the top of a big tree, which would otherwise be the serial fraction of the parallel
 * build: the range is cut into chunks binned concurrently, and the partial bins are merged IN CHUNK ORDER with the same
 * min/max macros.  Those macros return their second argument on ties, so a left-to-right fold and an ordered fold of
 * per-chunk folds pick the same element (this matters only for the sign of zero, +0 == -0); counts just add. */
#define PARALLEL_BIN_PRIMS 32768u
struct bin_job { const struct builder *B; const float *bounds; unsigned begin, end; int chunks; struct bin (*part)[3][BIN_COUNT]; };

static void bin_chunk(void *arg, int k) {
	struct bin_job *j = arg;
	const unsigned n = j->end - j->begin;
	const unsigned b = j->begin + (unsigned)((unsigned long long)n * (unsigned)k / (unsigned)j->chunks);
	const unsigned e = j->begin + (unsigned)((unsigned long long)n * (unsigned)(k + 1) / (unsigned)j->chunks);
	fill_bins(j->B, j->bounds, b, e, j->part[k]);
}

static void fill_bins_parallel(const struct builder *B, const float bounds[6], unsigned begin, unsigned end, struct bin bins[3][BIN_COUNT]) {
	int chunks = crl_thread_count();
	if (chunks > 64) chunks = 64;
	struct bin_job job = { B, bounds, begin, end, chunks, malloc(sizeof(struct bin) * 3 * BIN_COUNT * (size_t)chunks) };
	if (!job.part) { fill_bins(B, bounds, begin, end, bins); return; }
	crl_parallel_for(chunks, bin_chunk, &job);
	for (int axis = 0; axis < 3; ++axis)
		for (int i = 0; i < BIN_COUNT; ++i) {
			struct bin *d = &bins[axis][i];
			d->bbox = crl_empty_bbox; d->count = 0;
			for (int k = 0; k < chunks; ++k) { bbox_extend(&d->bbox, &job.part[k][axis][i].bbox); d->count += job.part[k][axis][i].count; }
		}
	free(job.part);
}

/* One node of the reference's buildBvhRecursive (bvh.c:137-243): decide leaf / split for prims[begin,end) inside
 * `bounds`; on a split the range is partitioned in place and the children's boxes are returned.  1 = split, 0 = leaf. */
static int split_node(const struct builder *B, const float bounds[6], unsigned begin, unsigned end, unsigned depth,
                      struct bin bins[3][BIN_COUNT], bbox3 *lb, bbox3 *rb, unsigned *beginRight) {
	const unsigned primCount = end - begin;
	if (depth >= MAX_DEPTH || primCount < 2) return 0;
	int32_t *prims = B->prims;
	float minCost[3] = { FLT_MAX, FLT_MAX, FLT_MAX };
	unsigned minBin[3] = { 1, 1, 1 };
	if (primCount >= PARALLEL_BIN_PRIMS && crl_thread_count() > 1) fill_bins_parallel(B, bounds, begin, end, bins);
	else fill_bins(B, bounds, begin, end, bins);
	for (int axis = 0; axis < 3; ++axis) {
		struct bin *ab = bins[axis];
		bbox3 cur = crl_empty_bbox;
		unsigned curCount = 0;
		for (unsigned i = BIN_COUNT; i > 1; --i) {                /* cost of everything to the right of a split */
			struct bin *b = &ab[i - 1];
			curCount += b->count;
			bbox_extend(&cur, &b->bbox);
			b->cost = curCount * bbox_half_area(&cur);
		}
		cur = crl_empty_bbox;
		curCount = 0;
		for (unsigned i = 0; i < BIN_COUNT - 1; i++) {
			struct bin *b = &ab[i];
			curCount += b->count;
			bbox_extend(&cur, &b->bbox);
			float cost = curCount * bbox_half_area(&cur) + ab[i + 1].cost;
			if (cost < minCost[axis]) { minBin[axis] = i + 1; minCost[axis] = cost; }
		}
	}
	unsigned minAxis = 0;
	if (minCost[1] < minCost[0]) minAxis = 1;
	if (minCost[2] < minCost[minAxis]) minAxis = 2;

	bbox3 nb = { { bounds[0], bounds[2], bounds[4] }, { bounds[1], bounds[3], bounds[5] } };
	float leafCost = bbox_half_area(&nb) * (primCount - TRAVERSAL_COST);
	if (minCost[minAxis] > leafCost) {
		if (primCount <= MAX_LEAF_SIZE) return 0;
		unsigned accum = 0, best = primCount;                     /* approximate median split (bvh.c:196-205) */
		for (unsigned i = 0; i < BIN_COUNT - 1; ++i) {
			accum += bins[minAxis][i].count;
			unsigned approx = (unsigned)abs((int)primCount / 2 - (int)accum);
			if (approx < best) { best = approx; minBin[minAxis] = i + 1; }
		}
	}

	/* two-pointer partition: everything in a bin below the split goes left (bvh.c:97-135) */
	const unsigned split = minBin[minAxis];
	const float lo = bounds[minAxis * 2], scale = BIN_COUNT / (bounds[minAxis * 2 + 1] - lo);
	unsigned i = begin, j = end;
	while (i < j) {
		while (i < j && bin_index(axis_of(&B->centers[prims[i]], (int)minAxis), lo, scale) < split) i++;
		while (i < j && bin_index(axis_of(&B->centers[prims[j - 1]], (int)minAxis), lo, scale) >= split) j--;
		if (i >= j) break;
		int32_t tmp = prims[j - 1]; prims[j - 1] = prims[i]; prims[i] = tmp;
		j--; i++;
	}
	if (i <= begin) return 0;
	*beginRight = i;
	*lb = crl_empty_bbox; *rb = crl_empty_bbox;
	for (unsigned k = 0; k < split; ++k) bbox_extend(lb, &bins[minAxis][k].bbox);
	for (unsigned k = split; k < BIN_COUNT; ++k) bbox_extend(rb, &bins[minAxis][k].bbox);
	return 1;
}

/* Serial build of one subtree into *nodes (room for *cap nodes, grown with realloc as needed): (*nodes)[0] is the subtree root
 * (bounds already stored), descendants are appended in the reference's allocation order (children as a pair when their parent is
 * visited, left subtree first).  Child links are indices into this local array.  Returns the number of nodes, 0 when out of memory.
 * A tree can need more than 2n-1 nodes: when every primitive of a node falls into bin 0 of the chosen axis (a zero extent, where the
 * bin scale is inf, or an extent that overflows to inf, where it is 0), every cost is NaN or inf and the split sends everything left,
 * so the node gets an empty right leaf and a left child with the same primitives and box, down to the depth cap. */
struct work { unsigned node, begin, end, depth; };

static unsigned build_subtree(const struct builder *B, struct crs_bvh_node **nodes, size_t *cap, unsigned begin, unsigned end, unsigned depth) {
	struct bin bins[3][BIN_COUNT];
	struct work stack[MAX_DEPTH + 2];
	unsigned node_count = 1;
	int sp = 0;
	stack[sp++] = (struct work){ 0, begin, end, depth };
	while (sp) {
		const struct work w = stack[--sp];
		bbox3 lb, rb;
		unsigned beginRight;
		if (!split_node(B, (*nodes)[w.node].bounds, w.begin, w.end, w.depth, bins, &lb, &rb, &beginRight)) {
			make_leaf(&(*nodes)[w.node], w.begin, w.end - w.begin);
			continue;
		}
		if ((size_t)node_count + 2 > *cap) {
			const size_t grown = 2 * *cap + 2;
			struct crs_bvh_node *p = realloc(*nodes, sizeof(**nodes) * grown);
			if (!p) return 0;
			*nodes = p; *cap = grown;
		}
		struct crs_bvh_node *node = &(*nodes)[w.node];
		const unsigned left = node_count, right = left + 1;
		node_count += 2;
		store_bbox(&(*nodes)[left], &lb);
		store_bbox(&(*nodes)[right], &rb);
		node->first_child_or_prim = left;
		node->prim_count_leaf = 0;
		/* the reference recurses left first, so the left subtree claims node indices first: push right, then left */
		stack[sp++] = (struct work){ right, beginRight, w.end, w.depth + 1 };
		stack[sp++] = (struct work){ left, w.begin, beginRight, w.depth + 1 };
	}
	return node_count;
}

/* ---- parallel driver ------------------------------------------------------------------------------------------
 * The top of the tree is split serially (largest open range first) until there are enough independent subtrees;
 * those are built by a small pthread pool into private arrays; a final depth-first walk lays everything out in the
 * order the serial recursion would have produced, so the result does not depend on the thread count. */
struct top { float bounds[6]; unsigned begin, end, depth; int left, right; int task; int leaf; };
struct task { unsigned begin, end, depth; float bounds[6]; struct crs_bvh_node *nodes; size_t cap; unsigned count; };
struct pool { const struct builder *B; struct task *tasks; int ntasks; int next; };

static void *pool_worker(void *arg) {
	struct pool *p = arg;
	for (;;) {
		int t = __atomic_fetch_add(&p->next, 1, __ATOMIC_RELAXED);
		if (t >= p->ntasks) return NULL;
		struct task *k = &p->tasks[t];
		memcpy(k->nodes[0].bounds, k->bounds, sizeof(k->bounds));
		k->count = build_subtree(p->B, &k->nodes, &k->cap, k->begin, k->end, k->depth);     /* 0: out of memory */
	}
}

static void layout(const struct top *tops, const struct task *tasks, int t, unsigned g, struct crs_bvh_node *out, unsigned *counter) {
	/* explicit stack: the top tree is at most a few hundred nodes deep in the worst case */
	struct item { int t; unsigned g; } *stack = malloc(sizeof(*stack) * 4096);
	int sp = 0, cap = 4096;
	stack[sp++] = (struct item){ t, g };
	while (sp) {
		struct item it = stack[--sp];
		const struct top *n = &tops[it.t];
		if (n->task >= 0) {
			const struct task *k = &tasks[n->task];
			const unsigned base = *counter;                     /* local index c >= 1 -> base + c - 1 */
			out[it.g] = k->nodes[0];
			if (!(out[it.g].prim_count_leaf & CRS_BVH_LEAF_BIT)) out[it.g].first_child_or_prim += base - 1;
			for (unsigned c = 1; c < k->count; ++c) {
				out[base + c - 1] = k->nodes[c];
				if (!(k->nodes[c].prim_count_leaf & CRS_BVH_LEAF_BIT)) out[base + c - 1].first_child_or_prim += base - 1;
			}
			*counter += k->count - 1;
		} else if (n->leaf) {
			memcpy(out[it.g].bounds, n->bounds, sizeof(n->bounds));
			make_leaf(&out[it.g], n->begin, n->end - n->begin);
		} else {
			const unsigned l = *counter;
			*counter += 2;
			memcpy(out[it.g].bounds, n->bounds, sizeof(n->bounds));
			out[it.g].first_child_or_prim = l;
			out[it.g].prim_count_leaf = 0;
			if (sp + 2 > cap) { cap *= 2; stack = realloc(stack, sizeof(*stack) * (size_t)cap); }
			stack[sp++] = (struct item){ n->right, l + 1 };
			stack[sp++] = (struct item){ n->left, l };
		}
	}
	free(stack);
}

#define PARALLEL_MIN_PRIMS 8192u     /* below this a single serial build is faster than starting threads */
#define TASK_MIN_PRIMS     2048u

/* an alternative builder for large inputs (crloader_set_bvh_builder): the device build of SURVEY 8(f1), wired in by libcrhost */
static crloader_bvh_builder g_builder;
static uint32_t g_builder_min;
void crloader_set_bvh_builder(crloader_bvh_builder fn, uint32_t min_prims) { g_builder = fn; g_builder_min = min_prims; }

static int build_with_hook(void *user, crl_bbox_fn fn, unsigned count,
                           struct crs_bvh_node **out_nodes, uint32_t *out_count, int32_t **out_prims) {
	float *bb = malloc(sizeof(float) * 6 * (size_t)count), *ct = malloc(sizeof(float) * 3 * (size_t)count);
	struct crs_bvh_node *nodes = calloc((size_t)2 * count, sizeof(*nodes));
	int32_t *prims = malloc(sizeof(int32_t) * (size_t)count);
	int rc = -1;
	if (bb && ct && nodes && prims) {
		for (unsigned i = 0; i < count; ++i) {
			bbox3 b; vec3 c;
			fn(user, i, &b, &c);
			bb[6 * (size_t)i] = b.min.x; bb[6 * (size_t)i + 1] = b.min.y; bb[6 * (size_t)i + 2] = b.min.z;
			bb[6 * (size_t)i + 3] = b.max.x; bb[6 * (size_t)i + 4] = b.max.y; bb[6 * (size_t)i + 5] = b.max.z;
			ct[3 * (size_t)i] = c.x; ct[3 * (size_t)i + 1] = c.y; ct[3 * (size_t)i + 2] = c.z;
		}
		uint32_t n = 0;
		rc = g_builder(bb, ct, count, nodes, &n, prims);
		if (rc == 0 && n >= 1) { *out_nodes = realloc(nodes, sizeof(*nodes) * n); *out_count = n; *out_prims = prims; nodes = NULL; prims = NULL; }
		else rc = -1;
	}
	free(bb); free(ct); free(nodes); free(prims);
	return rc;
}

int crl_build_bvh(void *user, crl_bbox_fn fn, unsigned count,
                  struct crs_bvh_node **out_nodes, uint32_t *out_count, int32_t **out_prims) {
	*out_nodes = NULL; *out_count = 0; *out_prims = NULL;
	if (count < 1) return 0;
	if (g_builder && count >= g_builder_min && build_with_hook(user, fn, count, out_nodes, out_count, out_prims) == 0) return 0;
	vec3 *centers = malloc(sizeof(vec3) * count);
	bbox3 *bboxes = malloc(sizeof(bbox3) * count);
	int32_t *prims = malloc(sizeof(int32_t) * count);
	size_t node_cap = (size_t)2 * count - 1;              /* enough for any tree without empty leaves; grown when needed */
	struct crs_bvh_node *nodes = calloc(node_cap, sizeof(*nodes));
	if (!centers || !bboxes || !prims || !nodes) { free(centers); free(bboxes); free(prims); free(nodes); return -1; }

	bbox3 root = crl_empty_bbox;
	for (unsigned i = 0; i < count; ++i) {
		fn(user, i, &bboxes[i], &centers[i]);
		prims[i] = (int32_t)i;
		root.min = v_min(root.min, bboxes[i].min);
		root.max = v_max(root.max, bboxes[i].max);
	}
	const struct builder B = { bboxes, centers, prims };
	unsigned node_count = 0;
	const int threads = crl_thread_count();
	if (threads < 2 || count < PARALLEL_MIN_PRIMS) {
		store_bbox(&nodes[0], &root);
		node_count = build_subtree(&B, &nodes, &node_cap, 0, count, 0);
		if (!node_count) { free(centers); free(bboxes); free(prims); free(nodes); return -1; }
	} else {
		/* 1. open the top of the tree serially, always splitting the largest open range */
		const int want = threads * 4;
		int ntops = 1, cap = 4 * want + 16, nopen = 1;
		struct top *tops = calloc((size_t)cap, sizeof(*tops));
		int *open = malloc(sizeof(int) * (size_t)cap);
		struct bin (*bins)[BIN_COUNT] = malloc(sizeof(struct bin) * 3 * BIN_COUNT);
		struct crs_bvh_node tmp;
		store_bbox(&tmp, &root);
		memcpy(tops[0].bounds, tmp.bounds, sizeof(tmp.bounds));
		tops[0] = (struct top){ .begin = 0, .end = count, .depth = 0, .left = -1, .right = -1, .task = -1 };
		memcpy(tops[0].bounds, tmp.bounds, sizeof(tmp.bounds));
		open[0] = 0;
		while (nopen < want && ntops + 2 <= cap) {
			int best = -1;
			for (int i = 0; i < nopen; ++i)
				if (best < 0 || tops[open[i]].end - tops[open[i]].begin > tops[open[best]].end - tops[open[best]].begin) best = i;
			struct top *n = &tops[open[best]];
			if (n->end - n->begin < TASK_MIN_PRIMS) break;
			open[best] = open[--nopen];
			bbox3 lb, rb;
			unsigned beginRight;
			if (!split_node(&B, n->bounds, n->begin, n->end, n->depth, bins, &lb, &rb, &beginRight)) { n->leaf = 1; continue; }
			n->left = ntops; n->right = ntops + 1;
			struct crs_bvh_node l, r;
			store_bbox(&l, &lb); store_bbox(&r, &rb);
			tops[ntops] = (struct top){ .begin = n->begin, .end = beginRight, .depth = n->depth + 1, .left = -1, .right = -1, .task = -1 };
			memcpy(tops[ntops].bounds, l.bounds, sizeof(l.bounds));
			tops[ntops + 1] = (struct top){ .begin = beginRight, .end = n->end, .depth = n->depth + 1, .left = -1, .right = -1, .task = -1 };
			memcpy(tops[ntops + 1].bounds, r.bounds, sizeof(r.bounds));
			open[nopen++] = ntops; open[nopen++] = ntops + 1;
			ntops += 2;
		}
		/* 2. every still-open range becomes a task, largest first */
		struct task *tasks = calloc((size_t)nopen + 1, sizeof(*tasks));
		for (int a = 0; a < nopen; ++a)
			for (int b = a + 1; b < nopen; ++b)
				if (tops[open[b]].end - tops[open[b]].begin > tops[open[a]].end - tops[open[a]].begin) { int t = open[a]; open[a] = open[b]; open[b] = t; }
		int ok = 1;
		for (int i = 0; i < nopen; ++i) {
			struct top *n = &tops[open[i]];
			n->task = i;
			tasks[i] = (struct task){ .begin = n->begin, .end = n->end, .depth = n->depth };
			memcpy(tasks[i].bounds, n->bounds, sizeof(n->bounds));
			tasks[i].cap = (size_t)2 * (n->end - n->begin) + 1;          /* an empty range (an empty right leaf) still has its root */
			tasks[i].nodes = calloc(tasks[i].cap, sizeof(struct crs_bvh_node));
			if (!tasks[i].nodes) ok = 0;
		}
		if (ok) {
			struct pool pool = { &B, tasks, nopen, 0 };
			int nthreads = threads < nopen ? threads : nopen;
			pthread_t *th = malloc(sizeof(pthread_t) * (size_t)nthreads);
			int started = 0;
			for (int i = 1; i < nthreads; ++i) if (pthread_create(&th[started], NULL, pool_worker, &pool) == 0) started++;
			pool_worker(&pool);
			for (int i = 0; i < started; ++i) pthread_join(th[i], NULL);
			free(th);
			/* 3. lay out in the serial recursion's order: every top node once, plus each task's nodes below its root */
			size_t total = (size_t)ntops;
			for (int i = 0; i < nopen; ++i) { if (!tasks[i].count) ok = 0; else total += tasks[i].count - 1; }
			if (ok && total > node_cap) {
				struct crs_bvh_node *p = realloc(nodes, sizeof(*nodes) * total);
				if (p) nodes = p; else ok = 0;
			}
			if (ok) {
				unsigned counter = 1;
				layout(tops, tasks, 0, 0, nodes, &counter);
				node_count = counter;
			}
		}
		for (int i = 0; i < nopen; ++i) free(tasks[i].nodes);
		free(tasks); free(tops); free(open); free(bins);
		if (!ok) { free(centers); free(bboxes); free(prims); free(nodes); return -1; }
	}
	free(centers); free(bboxes);
	*out_nodes = realloc(nodes, sizeof(*nodes) * node_count);
	*out_count = node_count;
	*out_prims = prims;
	return 0;
}

/* ---- the builder on its own (include/crloader.h) ---------------------------------------------------------------------------------- */
struct array_user { const float *bb, *ct; };
static void array_bbox(void *user, unsigned i, bbox3 *bbox, vec3 *center) {
	const struct array_user *u = user;
	bbox->min = (vec3){ u->bb[6 * (size_t)i], u->bb[6 * (size_t)i + 1], u->bb[6 * (size_t)i + 2] };
	bbox->max = (vec3){ u->bb[6 * (size_t)i + 3], u->bb[6 * (size_t)i + 4], u->bb[6 * (size_t)i + 5] };
	*center = (vec3){ u->ct[3 * (size_t)i], u->ct[3 * (size_t)i + 1], u->ct[3 * (size_t)i + 2] };
}

int crloader_build_bvh(const float *bboxes, const float *centers, uint32_t n,
                       struct crs_bvh_node *nodes_out, uint32_t *node_count_out, int32_t *prims_out) {
	if (!node_count_out || (n && (!bboxes || !centers || !nodes_out || !prims_out))) { crl_set_error("crloader_build_bvh: NULL argument"); return -1; }
	*node_count_out = 0;
	if (n == 0) return 0;
	struct array_user u = { bboxes, centers };
	struct crs_bvh_node *nodes = NULL;
	int32_t *prims = NULL;
	uint32_t cnt = 0;
	const crloader_bvh_builder saved = g_builder;
	g_builder = NULL;                                  /* always the host algorithm */
	const int rc = crl_build_bvh(&u, array_bbox, n, &nodes, &cnt, &prims);
	g_builder = saved;
	int out = rc;
	if (rc) crl_set_error("crloader_build_bvh: out of memory");
	if (rc == 0 && cnt > 2 * (uint64_t)n - 1) {          /* the caller has room for 2n-1 nodes: report the size, write nothing */
		*node_count_out = cnt;
		crl_set_error("crloader_build_bvh: the tree of %u primitives needs %u nodes, more than 2n - 1", n, cnt);
		out = -2;
	} else if (rc == 0) {
		memcpy(nodes_out, nodes, sizeof(*nodes) * cnt);
		memcpy(prims_out, prims, sizeof(int32_t) * n);
		*node_count_out = cnt;
	}
	free(nodes); free(prims);
	return out;
}
