/*
 * crgpu_bvh_build.cu — SURVEY §8(f1): the reference's binned-SAH BVH build on the device.
 *
 * Restates reference src/accelerators/bvh.c:96-296 (buildBvhRecursive + partitionPrimitives) so that the result is THE SAME tree
 * the reference (and host/loader/cr_bvh_build.c) builds — node for node, leaf range for leaf range, primitive order included —
 * because the traversal's tie-breaking depends on all three.  The recursion becomes a level-synchronous sweep: every open node of a
 * level is binned, split and partitioned by the same few kernels, whatever its size.
 *
 *   bins        the reference folds `bbox_extend` over a node's primitives in array order with the min/max MACROS (bvh.c:158-171);
 *               ties return the second operand, so the only order dependence is the SIGN OF ZERO of a bound, decided by the last
 *               tied primitive.  Here every bin bound is a 64-bit atomic min/max over (ordered value with -0 == +0, array position):
 *               the winner is the extreme value and, among ties, the last position; the float is then read back from that primitive.
 *   split       one thread per open node runs the two 32-bin sweeps of the three axes, the leaf-cost test and the approximate
 *               median fallback with the reference's float association (explicit __f*_rn: no contraction).
 *   partition   the reference's two-pointer in-place partition (bvh.c:97-135) swaps the k-th misplaced element from the left
 *               with the k-th misplaced element from the right; the ranks come from two prefix sums over the whole array.
 *   numbering   children are allocated as a pair when their parent is visited, left subtree first (bvh.c:221-239), i.e. the pair
 *               of internal node X sits at 1 + 2 * (number of internal nodes before X in left-first preorder): one bottom-up pass
 *               for subtree sizes, one top-down pass for the ranks.
 *
 * Float->unsigned conversions follow x86-64 cvttss2si like the host builder (f2u).  NaN coordinates are not supported (the
 * reference's own comparisons make the tree undefined there).  Limits: 4,194,304 primitives per call (two-level prefix sum).
 */
#include "../../include/crgpu.h"
#include "../../include/crscene.h"
#include "crgpu_bvh_build.cuh"
#include <cuda_runtime.h>
#include <stdint.h>
#include <string.h>
#include <utility>
#include <vector>

int crg_fail(int code, const char *fmt, ...);           /* crgpu_api.cu: sets crgpu_last_error() */

#define BVB_BINS 32
#define BVB_MAX_DEPTH 64u
#define BVB_MAX_LEAF 16u
#define BVB_SCAN_BLOCK 1024u     /* elements per scan block: 256 threads x 4 */
#define BVB_FLT_MAX 3.402823466e+38f

namespace {

struct Rec {                     /* one per tree node, in creation order (levels are contiguous) */
	uint32_t begin, end, depth;
	int32_t  left;               /* record of the left child (right = left + 1); -1 leaf; -2 open (to be decided) */
	float    b[6];               /* minx,maxx,miny,maxy,minz,maxz */
	uint32_t axis, split, mid;   /* split decision of an internal node; mid = first position of the right child */
	uint32_t slot;               /* index among the open nodes of its level */
	uint32_t internals, rank, idx;
	float    lb[6], rb[6];       /* children's bounds (bvh.c:210-217) */
};

struct Bins {                    /* per open node of the current level */
	unsigned           cnt[3][BVB_BINS];
	unsigned long long kmin[3][BVB_BINS][3];
	unsigned long long kmax[3][BVB_BINS][3];
};

__device__ __forceinline__ uint32_t okey(float f) {
	f = __fadd_rn(f, 0.0f);                              /* -0 -> +0: equal values must have equal keys */
	const uint32_t b = __float_as_uint(f);
	return (b & 0x80000000u) ? ~b : (b | 0x80000000u);
}
__device__ __forceinline__ unsigned long long key_max(float f, uint32_t pos) { return ((unsigned long long)okey(f) << 32) | pos; }
__device__ __forceinline__ unsigned long long key_min(float f, uint32_t pos) { return ((unsigned long long)okey(f) << 32) | (uint32_t)~pos; }
#define KMIN_EMPTY 0xffffffffffffffffull
#define KMAX_EMPTY 0ull

/* (unsigned)f as GCC compiles it on x86-64 (cvttss2si to 64 bits, low half kept), cr_bvh_build.c f2u */
__device__ __forceinline__ unsigned f2u(float f) {
	if (!(f > -9.2233720e18f && f < 9.2233720e18f)) return 0u;
	return (unsigned)(unsigned long long)__float2ll_rz(f);
}
__device__ __forceinline__ unsigned bin_index(float coord, float lo, float scale) {         /* bvh.c:89-95 */
	const float fi = __fmul_rn(__fsub_rn(coord, lo), scale);
	const unsigned b = f2u(fi < 0 ? 0 : fi);
	return b >= BVB_BINS ? BVB_BINS - 1 : b;
}
__device__ __forceinline__ float bin_scale(const float *b, int axis) { return __fdiv_rn((float)BVB_BINS, __fsub_rn(b[2 * axis + 1], b[2 * axis])); }
__device__ __forceinline__ float half_area(const float *mn, const float *mx) {               /* bbox.h:26 */
	const float ex = __fsub_rn(mx[0], mn[0]), ey = __fsub_rn(mx[1], mn[1]), ez = __fsub_rn(mx[2], mn[2]);
	return __fadd_rn(__fmul_rn(ex, __fadd_rn(ey, ez)), __fmul_rn(ey, ez));
}
#define MACRO_MIN(a, b) ((a) < (b) ? (a) : (b))
#define MACRO_MAX(a, b) ((a) > (b) ? (a) : (b))

/* ---- root bounds: the fold of bvh.c:266-271 over all primitives in order ------------------------------------------------------- */
__global__ void k_root_keys(const float *__restrict__ bb, uint32_t n, unsigned long long *keys /* [6]: min xyz, max xyz */) {
	const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
	if (i >= n) return;
	for (int k = 0; k < 3; ++k) {
		atomicMin(&keys[k], key_min(bb[6 * (size_t)i + k], i));
		atomicMax(&keys[3 + k], key_max(bb[6 * (size_t)i + 3 + k], i));
	}
}
__global__ void k_root_init(const float *__restrict__ bb, uint32_t n, const unsigned long long *keys, Rec *recs, uint32_t *counters) {
	Rec r;
	memset(&r, 0, sizeof r);
	r.begin = 0u; r.end = n; r.depth = 0u; r.slot = 0u;
	for (int k = 0; k < 3; ++k) {
		const uint32_t pmin = ~(uint32_t)(keys[k] & 0xffffffffull), pmax = (uint32_t)(keys[3 + k] & 0xffffffffull);
		r.b[2 * k] = bb[6 * (size_t)pmin + k];
		r.b[2 * k + 1] = bb[6 * (size_t)pmax + 3 + k];
	}
	const bool open = n >= 2u;
	r.left = open ? -2 : -1;
	recs[0] = r;
	counters[0] = 1u;                  /* records allocated */
	counters[1] = open ? 1u : 0u;      /* open nodes of the current level */
	counters[2] = 0u;                  /* open nodes of the next level */
}

/* ---- bins (bvh.c:158-171) ------------------------------------------------------------------------------------------------------- */
__global__ void k_bin(const float *__restrict__ bb, const float *__restrict__ ctr, const int32_t *__restrict__ prims,
					  const int32_t *__restrict__ owner, const Rec *__restrict__ recs, Bins *bins, uint32_t n) {
	const uint32_t pos = blockIdx.x * blockDim.x + threadIdx.x;
	if (pos >= n) return;
	const int32_t r = owner[pos];
	if (r < 0) return;
	const Rec &rec = recs[r];
	Bins &B = bins[rec.slot];
	const uint32_t p = (uint32_t)prims[pos];
	const float *pb = bb + 6 * (size_t)p;
	for (int axis = 0; axis < 3; ++axis) {
		const unsigned bi = bin_index(ctr[3 * (size_t)p + axis], rec.b[2 * axis], bin_scale(rec.b, axis));
		atomicAdd(&B.cnt[axis][bi], 1u);
		for (int k = 0; k < 3; ++k) {
			atomicMin(&B.kmin[axis][bi][k], key_min(pb[k], pos));
			atomicMax(&B.kmax[axis][bi][k], key_max(pb[3 + k], pos));
		}
	}
}
__global__ void k_bins_clear(Bins *bins, uint32_t count) {
	const size_t words = (size_t)count * (sizeof(Bins) / 8u);
	unsigned long long *w = reinterpret_cast<unsigned long long *>(bins);
	for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < words; i += (size_t)gridDim.x * blockDim.x) {
		const size_t in = i % (sizeof(Bins) / 8u);
		const size_t cnt_words = sizeof(unsigned) * 3 * BVB_BINS / 8u, key_words = 3u * BVB_BINS * 3u;
		w[i] = in < cnt_words ? 0ull : (in < cnt_words + key_words ? KMIN_EMPTY : KMAX_EMPTY);
	}
}

/* ---- split decision: bvh.c:137-207, one thread per open node --------------------------------------------------------------------- */
__global__ void k_split(const float *__restrict__ bb, const int32_t *__restrict__ prims, Rec *recs, const uint32_t *__restrict__ open_list,
						uint32_t nopen, const Bins *__restrict__ bins) {
	const uint32_t s = blockIdx.x * blockDim.x + threadIdx.x;
	if (s >= nopen) return;
	Rec &rec = recs[open_list[s]];
	const Bins &B = bins[s];
	const uint32_t primCount = rec.end - rec.begin;
	float bmin[BVB_BINS][3], bmax[BVB_BINS][3], bcost[BVB_BINS];
	float minCost[3] = { BVB_FLT_MAX, BVB_FLT_MAX, BVB_FLT_MAX };
	unsigned minBin[3] = { 1u, 1u, 1u };
	float bestLb[6], bestRb[6];
	unsigned minAxis = 0u;
	/* the sweeps of the three axes; the bins of the winning axis are needed again for the children's boxes, so the axis loop runs
	 * once to find the winner and the winner's bins are resolved a second time below (cheaper than keeping 3 x 32 boxes) */
	for (int pass = 0; pass < 2; ++pass) {
		for (int axis = 0; axis < 3; ++axis) {
			if (pass == 1 && (unsigned)axis != minAxis) continue;
			for (int i = 0; i < BVB_BINS; ++i)
				for (int k = 0; k < 3; ++k) {
					const unsigned long long a = B.kmin[axis][i][k], c = B.kmax[axis][i][k];
					bmin[i][k] = a == KMIN_EMPTY ? BVB_FLT_MAX : bb[6 * (size_t)prims[~(uint32_t)(a & 0xffffffffull)] + k];
					bmax[i][k] = c == KMAX_EMPTY ? -BVB_FLT_MAX : bb[6 * (size_t)prims[(uint32_t)(c & 0xffffffffull)] + 3 + k];
				}
			if (pass == 1) break;
			float cmin[3] = { BVB_FLT_MAX, BVB_FLT_MAX, BVB_FLT_MAX }, cmax[3] = { -BVB_FLT_MAX, -BVB_FLT_MAX, -BVB_FLT_MAX };
			unsigned curCount = 0u;
			for (unsigned i = BVB_BINS; i > 1; --i) {                  /* cost of everything to the right of a split */
				curCount += B.cnt[axis][i - 1];
				for (int k = 0; k < 3; ++k) { cmin[k] = MACRO_MIN(cmin[k], bmin[i - 1][k]); cmax[k] = MACRO_MAX(cmax[k], bmax[i - 1][k]); }
				bcost[i - 1] = __fmul_rn(__uint2float_rn(curCount), half_area(cmin, cmax));
			}
			for (int k = 0; k < 3; ++k) { cmin[k] = BVB_FLT_MAX; cmax[k] = -BVB_FLT_MAX; }
			curCount = 0u;
			for (unsigned i = 0; i < BVB_BINS - 1; ++i) {
				curCount += B.cnt[axis][i];
				for (int k = 0; k < 3; ++k) { cmin[k] = MACRO_MIN(cmin[k], bmin[i][k]); cmax[k] = MACRO_MAX(cmax[k], bmax[i][k]); }
				const float cost = __fadd_rn(__fmul_rn(__uint2float_rn(curCount), half_area(cmin, cmax)), bcost[i + 1]);
				if (cost < minCost[axis]) { minBin[axis] = i + 1; minCost[axis] = cost; }
			}
		}
		if (pass == 0) {
			minAxis = 0u;
			if (minCost[1] < minCost[0]) minAxis = 1u;
			if (minCost[2] < minCost[minAxis]) minAxis = 2u;
		}
	}
	const float nmin[3] = { rec.b[0], rec.b[2], rec.b[4] }, nmax[3] = { rec.b[1], rec.b[3], rec.b[5] };
	const float leafCost = __fmul_rn(half_area(nmin, nmax), __fsub_rn(__uint2float_rn(primCount), 1.5f));
	if (minCost[minAxis] > leafCost) {
		if (primCount <= BVB_MAX_LEAF) { rec.left = -1; return; }
		unsigned accum = 0u, best = primCount;                        /* approximate median split (bvh.c:196-205) */
		for (unsigned i = 0; i < BVB_BINS - 1; ++i) {
			accum += B.cnt[minAxis][i];
			const int dlt = (int)primCount / 2 - (int)accum;
			const unsigned approx = (unsigned)(dlt < 0 ? -dlt : dlt);
			if (approx < best) { best = approx; minBin[minAxis] = i + 1; }
		}
	}
	const unsigned split = minBin[minAxis];
	for (int k = 0; k < 3; ++k) { bestLb[2 * k] = BVB_FLT_MAX; bestLb[2 * k + 1] = -BVB_FLT_MAX; bestRb[2 * k] = BVB_FLT_MAX; bestRb[2 * k + 1] = -BVB_FLT_MAX; }
	for (unsigned i = 0; i < split; ++i)
		for (int k = 0; k < 3; ++k) { bestLb[2 * k] = MACRO_MIN(bestLb[2 * k], bmin[i][k]); bestLb[2 * k + 1] = MACRO_MAX(bestLb[2 * k + 1], bmax[i][k]); }
	for (unsigned i = split; i < BVB_BINS; ++i)
		for (int k = 0; k < 3; ++k) { bestRb[2 * k] = MACRO_MIN(bestRb[2 * k], bmin[i][k]); bestRb[2 * k + 1] = MACRO_MAX(bestRb[2 * k + 1], bmax[i][k]); }
	rec.axis = minAxis; rec.split = split;
	for (int k = 0; k < 6; ++k) { rec.lb[k] = bestLb[k]; rec.rb[k] = bestRb[k]; }
	/* rec.left stays -2: the partition decides whether anything goes left (bvh.c:229) */
}

/* ---- partition (bvh.c:97-135) ---------------------------------------------------------------------------------------------------- */
__global__ void k_flag(const float *__restrict__ ctr, const int32_t *__restrict__ prims, const int32_t *__restrict__ owner,
					   const Rec *__restrict__ recs, unsigned long long *flags, uint32_t n) {
	const uint32_t pos = blockIdx.x * blockDim.x + threadIdx.x;
	if (pos >= n) return;
	unsigned long long f = 0ull;
	const int32_t r = owner[pos];
	if (r >= 0 && recs[r].left == -2) {
		const Rec &rec = recs[r];
		const int axis = (int)rec.axis;
		f = bin_index(ctr[3 * (size_t)prims[pos] + axis], rec.b[2 * axis], bin_scale(rec.b, axis)) < rec.split ? 1ull : 0ull;
	}
	flags[pos] = f;
}
__global__ void k_mid(Rec *recs, const uint32_t *__restrict__ open_list, uint32_t nopen, const unsigned long long *__restrict__ S1) {
	const uint32_t s = blockIdx.x * blockDim.x + threadIdx.x;
	if (s >= nopen) return;
	Rec &rec = recs[open_list[s]];
	if (rec.left != -2) return;
	const unsigned long long before = rec.begin ? S1[rec.begin - 1u] : 0ull;
	rec.mid = rec.begin + (uint32_t)(S1[rec.end - 1u] - before);
	if (rec.mid <= rec.begin) rec.left = -1;                           /* bvh.c:229: nothing went left -> leaf */
}
/* misplaced elements: low half = flag-0 elements left of mid, high half = flag-1 elements right of mid */
__global__ void k_misplaced(const int32_t *__restrict__ owner, const Rec *__restrict__ recs, const unsigned long long *__restrict__ flags,
							unsigned long long *mis, uint32_t n) {
	const uint32_t pos = blockIdx.x * blockDim.x + threadIdx.x;
	if (pos >= n) return;
	unsigned long long m = 0ull;
	const int32_t r = owner[pos];
	if (r >= 0 && recs[r].left == -2) {
		const bool fl = flags[pos] != 0ull;
		if (pos < recs[r].mid) { if (!fl) m = 1ull; } else if (fl) m = 1ull << 32;
	}
	mis[pos] = m;
}
__global__ void k_scatter_right(const int32_t *__restrict__ owner, const Rec *__restrict__ recs, const unsigned long long *__restrict__ mis,
								const unsigned long long *__restrict__ S2, uint32_t *tmpR, uint32_t n) {
	const uint32_t pos = blockIdx.x * blockDim.x + threadIdx.x;
	if (pos >= n || !(mis[pos] >> 32)) return;
	const Rec &rec = recs[owner[pos]];
	const uint32_t rankR = (uint32_t)(S2[rec.end - 1u] >> 32) - (uint32_t)(S2[pos] >> 32);     /* 0 = the rightmost one */
	tmpR[rec.begin + rankR] = pos;
}
__global__ void k_swap(const int32_t *__restrict__ owner, const Rec *__restrict__ recs, const unsigned long long *__restrict__ mis,
					   const unsigned long long *__restrict__ S2, const uint32_t *__restrict__ tmpR, int32_t *prims, uint32_t n) {
	const uint32_t pos = blockIdx.x * blockDim.x + threadIdx.x;
	if (pos >= n || !(mis[pos] & 0xffffffffull)) return;
	const Rec &rec = recs[owner[pos]];
	const uint32_t before = rec.begin ? (uint32_t)(S2[rec.begin - 1u] & 0xffffffffull) : 0u;
	const uint32_t k = (uint32_t)(S2[pos] & 0xffffffffull) - before - 1u;                        /* 0 = the leftmost one */
	const uint32_t partner = tmpR[rec.begin + k];
	const int32_t a = prims[pos], b = prims[partner];
	prims[pos] = b; prims[partner] = a;
}

/* ---- children (bvh.c:221-239) ----------------------------------------------------------------------------------------------------- */
__global__ void k_children(Rec *recs, const uint32_t *__restrict__ open_list, uint32_t nopen, uint32_t *next_list, uint32_t *counters) {
	const uint32_t s = blockIdx.x * blockDim.x + threadIdx.x;
	if (s >= nopen) return;
	const uint32_t ri = open_list[s];
	Rec &rec = recs[ri];
	if (rec.left != -2) return;
	const uint32_t c = atomicAdd(&counters[0], 2u);
	rec.left = (int32_t)c;
	for (int side = 0; side < 2; ++side) {
		Rec ch;
		memset(&ch, 0, sizeof ch);
		ch.begin = side ? rec.mid : rec.begin;
		ch.end = side ? rec.end : rec.mid;
		ch.depth = rec.depth + 1u;
		for (int k = 0; k < 6; ++k) ch.b[k] = side ? rec.rb[k] : rec.lb[k];
		const bool open = ch.depth < BVB_MAX_DEPTH && ch.end - ch.begin >= 2u;     /* bvh.c:138-141 */
		ch.left = open ? -2 : -1;
		if (open) { ch.slot = atomicAdd(&counters[2], 1u); next_list[ch.slot] = c + (uint32_t)side; }
		recs[c + side] = ch;
	}
}
__global__ void k_owner(int32_t *owner, const Rec *__restrict__ recs, uint32_t n) {
	const uint32_t pos = blockIdx.x * blockDim.x + threadIdx.x;
	if (pos >= n) return;
	const int32_t r = owner[pos];
	if (r < 0) return;
	const Rec &rec = recs[r];
	int32_t o = -1;
	if (rec.left >= 0) {
		const int32_t child = rec.left + (pos < rec.mid ? 0 : 1);
		if (recs[child].left == -2) o = child;
	}
	owner[pos] = o;
}
__global__ void k_level_advance(uint32_t *counters) { counters[1] = counters[2]; counters[2] = 0u; }

/* ---- numbering ------------------------------------------------------------------------------------------------------------------------ */
__global__ void k_count_internals(Rec *recs, uint32_t first, uint32_t count) {
	const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
	if (i >= count) return;
	Rec &r = recs[first + i];
	r.internals = r.left >= 0 ? 1u + recs[r.left].internals + recs[r.left + 1].internals : 0u;
}
__global__ void k_assign(Rec *recs, uint32_t first, uint32_t count) {
	const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
	if (i >= count) return;
	const Rec &r = recs[first + i];
	if (r.left < 0) return;
	Rec &l = recs[r.left], &rr = recs[r.left + 1];
	l.rank = r.rank + 1u; rr.rank = r.rank + 1u + l.internals;
	l.idx = 1u + 2u * r.rank; rr.idx = 2u + 2u * r.rank;
}
__global__ void k_emit(const Rec *__restrict__ recs, uint32_t nrec, crs_bvh_node *out) {
	const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
	if (i >= nrec) return;
	const Rec &r = recs[i];
	crs_bvh_node nd;
	for (int k = 0; k < 6; ++k) nd.bounds[k] = r.b[k];
	if (r.left >= 0) { nd.first_child_or_prim = 1u + 2u * r.rank; nd.prim_count_leaf = 0u; }
	else { nd.first_child_or_prim = r.begin; nd.prim_count_leaf = CRS_BVH_LEAF_BIT | ((r.end - r.begin) & CRS_BVH_COUNT_MASK); }
	out[r.idx] = nd;
}
__global__ void k_iota(int32_t *prims, int32_t *owner, uint32_t n, int32_t owner0) {
	const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
	if (i < n) { prims[i] = (int32_t)i; owner[i] = owner0; }
}

/* ---- inclusive prefix sum of 64-bit words (both halves at once: the halves never carry into each other, counts < 2^32) ------------- */
__global__ void __launch_bounds__(256) k_scan_blocks(const unsigned long long *__restrict__ in, unsigned long long *out, unsigned long long *sums, uint32_t n) {
	__shared__ unsigned long long s_warp[8];
	const uint32_t base = blockIdx.x * BVB_SCAN_BLOCK + threadIdx.x * 4u;
	unsigned long long v[4], acc = 0ull;
	for (int k = 0; k < 4; ++k) { v[k] = base + k < n ? in[base + k] : 0ull; acc += v[k]; v[k] = acc; }
	unsigned long long incl = acc;
	const unsigned lane = threadIdx.x & 31u, w = threadIdx.x >> 5;
	for (unsigned d = 1; d < 32; d <<= 1) { const unsigned long long x = __shfl_up_sync(0xffffffffu, incl, d); if (lane >= d) incl += x; }
	if (lane == 31u) s_warp[w] = incl;
	__syncthreads();
	unsigned long long woff = 0ull;
	for (unsigned k = 0; k < w; ++k) woff += s_warp[k];
	const unsigned long long excl = woff + incl - acc;
	for (int k = 0; k < 4; ++k) if (base + k < n) out[base + k] = excl + v[k];
	if (threadIdx.x == 255u && sums) sums[blockIdx.x] = woff + incl;
}
__global__ void k_scan_add(unsigned long long *out, const unsigned long long *__restrict__ sums_incl, uint32_t n) {
	const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
	const uint32_t blk = i / BVB_SCAN_BLOCK;
	if (i < n && blk > 0u) out[i] += sums_incl[blk - 1u];
}

/* ---- the pair layout of an edited scene's BVHs, top level or mesh (crgpu_api.cu build_pairs, on the device) ------------------------
 * build_pairs numbers internal nodes in BFS order, children left before right.  Records are created level by level, but in atomic
 * order within a level, so one block walks the levels in BFS order: per level, an exclusive block scan of the internal-child counts
 * of the level's internal nodes (in their BFS order) places their internal children in the next level. */
__global__ void __launch_bounds__(1024) k_pair_bfs(const Rec *__restrict__ recs, uint32_t *order, uint32_t *bfs_of, uint32_t *info) {
	__shared__ uint32_t s_warp[32];
	const unsigned lane = threadIdx.x & 31u, w = threadIdx.x >> 5, nw = blockDim.x >> 5;
	if (threadIdx.x == 0) { order[0] = 0u; bfs_of[0] = 0u; }
	__syncthreads();
	uint32_t lo = 0u, hi = 1u, tail = 1u, levels = 0u;
	while (lo < hi) {
		++levels;
		for (uint32_t base = lo; base < hi; base += blockDim.x) {
			const uint32_t j = base + threadIdx.x;
			int32_t L = -1;
			bool il = false, ir = false;
			if (j < hi) { L = recs[order[j]].left; il = recs[L].left >= 0; ir = recs[L + 1].left >= 0; }
			const uint32_t c = (il ? 1u : 0u) + (ir ? 1u : 0u);
			uint32_t incl = c;
			for (unsigned d = 1; d < 32; d <<= 1) { const uint32_t x = __shfl_up_sync(0xffffffffu, incl, d); if (lane >= d) incl += x; }
			if (lane == 31u) s_warp[w] = incl;
			__syncthreads();
			uint32_t woff = 0u, total = 0u;
			for (unsigned k = 0; k < nw; ++k) { if (k < w) woff += s_warp[k]; total += s_warp[k]; }
			if (j < hi) {
				uint32_t p = tail + woff + incl - c;
				if (il) { order[p] = (uint32_t)L; bfs_of[L] = p; ++p; }
				if (ir) { order[p] = (uint32_t)L + 1u; bfs_of[L + 1] = p; }
			}
			tail += total;
			__syncthreads();                 /* s_warp is reused; the next level reads what this one wrote */
		}
		lo = hi; hi = tail;
	}
	if (threadIdx.x == 0) { info[0] = tail; info[1] = levels; }
}
__global__ void k_pairs(const Rec *__restrict__ recs, const uint32_t *__restrict__ order, const uint32_t *__restrict__ bfs_of, uint32_t count,
							PairNode *pairs) {
	const uint32_t r = blockIdx.x * blockDim.x + threadIdx.x;
	if (r >= count) return;
	const Rec &R = recs[order[r]];
	PairNode p;
	for (int side = 0; side < 2; ++side) {
		const int32_t ci = R.left + side;
		const Rec &c = recs[ci];
		float *b = side ? p.rb : p.lb;
		for (int k = 0; k < 6; ++k) b[k] = c.b[k];
		const uint32_t ref = c.left >= 0 ? bfs_of[ci] : c.begin, meta = c.left >= 0 ? 0u : CRG_LEAF_BIT | ((c.end - c.begin) & CRS_BVH_COUNT_MASK);
		if (side) { p.rref = ref; p.rmeta = meta; } else { p.lref = ref; p.lmeta = meta; }
	}
	pairs[r] = p;
}

/* the scratch of one build of n primitives, carved from one block (base == nullptr: only the size) */
struct Scratch {
	int32_t *prims, *owner;
	Rec *recs;
	Bins *bins;
	uint32_t *open[2], *tmpR, *cnt, *order, *bfs_of, *info;
	unsigned long long *flags, *S1, *mis, *S2, *sums, *sums2, *keys;
};
size_t carve(void *base, uint32_t n, Scratch *s) {
	const size_t max_open = n / 2u + 1u, max_rec = 2u * (size_t)n;
	size_t off = 0;
	auto take = [&](size_t bytes) { void *p = base ? static_cast<uint8_t *>(base) + off : nullptr; off += (bytes + 255u) & ~(size_t)255u; return p; };
	s->prims = (int32_t *)take((size_t)n * 4u); s->owner = (int32_t *)take((size_t)n * 4u);
	s->recs = (Rec *)take(max_rec * sizeof(Rec)); s->bins = (Bins *)take(max_open * sizeof(Bins));
	s->open[0] = (uint32_t *)take(max_open * 4u); s->open[1] = (uint32_t *)take(max_open * 4u);
	s->flags = (unsigned long long *)take((size_t)n * 8u); s->S1 = (unsigned long long *)take((size_t)n * 8u);
	s->mis = (unsigned long long *)take((size_t)n * 8u); s->S2 = (unsigned long long *)take((size_t)n * 8u);
	s->tmpR = (uint32_t *)take((size_t)n * 4u); s->sums = (unsigned long long *)take(8u * ((size_t)n / BVB_SCAN_BLOCK + 2u));
	s->sums2 = (unsigned long long *)take(8u * 64u); s->keys = (unsigned long long *)take(6u * 8u); s->cnt = (uint32_t *)take(4u * 4u);
	s->order = (uint32_t *)take((size_t)n * 4u); s->bfs_of = (uint32_t *)take(max_rec * 4u); s->info = (uint32_t *)take(4u * 4u);
	return off;
}

struct DevBuf {
	void *p = nullptr;
	~DevBuf() { if (p) cudaFree(p); }
	cudaError_t alloc(size_t bytes) { return cudaMalloc(&p, bytes ? bytes : 1); }
	template <class T> T *as() { return static_cast<T *>(p); }
};

}  // namespace

#define CUB(call) do { cudaError_t e_ = (call); if (e_ != cudaSuccess) return crg_fail(e_ == cudaErrorMemoryAllocation ? CRGPU_ERR_NOMEM : CRGPU_ERR_CUDA, "crgpu_bvh_build: %s: %s", #call, cudaGetErrorString(e_)); } while (0)

int crg_scan64(const unsigned long long *in, unsigned long long *out, unsigned long long *sums, unsigned long long *sums2, uint32_t n, cudaStream_t st) {
	const uint32_t nb = (n + BVB_SCAN_BLOCK - 1u) / BVB_SCAN_BLOCK;
	k_scan_blocks<<<nb, 256, 0, st>>>(in, out, sums, n);
	if (nb > 1u) {
		const uint32_t nb2 = (nb + BVB_SCAN_BLOCK - 1u) / BVB_SCAN_BLOCK;        /* <= 4 for n <= 4M */
		k_scan_blocks<<<nb2, 256, 0, st>>>(sums, sums, sums2, nb);
		if (nb2 > 1u) {
			k_scan_blocks<<<1, 256, 0, st>>>(sums2, sums2, nullptr, nb2);
			k_scan_add<<<(nb + 255u) / 256u, 256, 0, st>>>(sums, sums2, nb);
		}
		k_scan_add<<<(n + 255u) / 256u, 256, 0, st>>>(out, sums, n);
		return nb2 > 1u ? 5 : 3;
	}
	return 1;
}

/* The records of a build: the scratch's 2n until a level could need more, then a device array of their own.  A tree needs more than
 * 2n - 1 nodes only with empty leaves: when every primitive of a node falls into bin 0 of the chosen axis (zero extent: the bin scale
 * is inf; an extent that overflows: it is 0), every cost is NaN or inf and the split sends everything left, so the node gets an empty
 * right leaf and a left child with its primitives and box, down to the depth cap. */
struct RecStore {
	Rec *recs;
	size_t cap;
	DevBuf own;
};

/* The tree of n >= 1 primitives (device boxes and centres) into the scratch s, on st: records level by level in rs.recs, primitive
 * order in s.prims.  Synchronises st once per level (the open-node count sizes the next launches); a level adds at most two records
 * per open node, and the records grow before a level that could pass their end. */
static int build_tree(const float *bb, const float *ctr, uint32_t n, const Scratch &s, cudaStream_t st, RecStore &rs,
					  std::vector<uint32_t> &level_first, std::vector<uint32_t> &level_count, uint32_t *nrec_out) {
	const uint32_t max_open = n / 2u + 1u;
	const unsigned long long init_keys[6] = { KMIN_EMPTY, KMIN_EMPTY, KMIN_EMPTY, KMAX_EMPTY, KMAX_EMPTY, KMAX_EMPTY };
	CUB(cudaMemcpyAsync(s.keys, init_keys, sizeof init_keys, cudaMemcpyHostToDevice, st));
	const uint32_t gn = (n + 255u) / 256u;
	rs.recs = s.recs;
	rs.cap = 2u * (size_t)n;
	Rec *recs = rs.recs;
	uint32_t *counters = s.cnt;
	k_iota<<<gn, 256, 0, st>>>(s.prims, s.owner, n, n >= 2u ? 0 : -1);
	k_root_keys<<<gn, 256, 0, st>>>(bb, n, s.keys);
	k_root_init<<<1, 1, 0, st>>>(bb, n, s.keys, recs, counters);
	const uint32_t zero = 0u;
	CUB(cudaMemcpyAsync(s.open[0], &zero, 4u, cudaMemcpyHostToDevice, st));          /* the root is open node 0 of level 0 */
	level_first.assign(1, 0u);
	level_count.assign(1, 1u);
	uint32_t h[4] = { 1u, n >= 2u ? 1u : 0u, 0u, 0u };
	int cur = 0;
	while (h[1] > 0u) {
		const uint32_t nopen = h[1], go = (nopen + 127u) / 128u;
		if (nopen > max_open) return crg_fail(CRGPU_ERR_CUDA, "crgpu_bvh_build: %u open nodes for %u primitives", nopen, n);
		const size_t need = (size_t)h[0] + 2u * (size_t)nopen;
		if (need > rs.cap) {
			const size_t cap = need > 2u * rs.cap ? need : 2u * rs.cap;
			DevBuf grown;
			CUB(grown.alloc(cap * sizeof(Rec)));
			CUB(cudaMemcpyAsync(grown.p, recs, (size_t)h[0] * sizeof(Rec), cudaMemcpyDeviceToDevice, st));
			CUB(cudaStreamSynchronize(st));
			std::swap(rs.own.p, grown.p);                                   /* the previous own array (if any) is freed here */
			rs.recs = recs = rs.own.as<Rec>();
			rs.cap = cap;
		}
		uint32_t *open_list = s.open[cur], *next_list = s.open[cur ^ 1];
		{
			const size_t blocks = ((size_t)nopen * (sizeof(Bins) / 8u) + 255u) / 256u;          /* grid-stride loop inside */
			k_bins_clear<<<(unsigned)(blocks > 65535u ? 65535u : blocks), 256, 0, st>>>(s.bins, nopen);
		}
		k_bin<<<gn, 256, 0, st>>>(bb, ctr, s.prims, s.owner, recs, s.bins, n);
		k_split<<<go, 128, 0, st>>>(bb, s.prims, recs, open_list, nopen, s.bins);
		k_flag<<<gn, 256, 0, st>>>(ctr, s.prims, s.owner, recs, s.flags, n);
		crg_scan64(s.flags, s.S1, s.sums, s.sums2, n, st);
		k_mid<<<go, 128, 0, st>>>(recs, open_list, nopen, s.S1);
		k_misplaced<<<gn, 256, 0, st>>>(s.owner, recs, s.flags, s.mis, n);
		crg_scan64(s.mis, s.S2, s.sums, s.sums2, n, st);
		k_scatter_right<<<gn, 256, 0, st>>>(s.owner, recs, s.mis, s.S2, s.tmpR, n);
		k_swap<<<gn, 256, 0, st>>>(s.owner, recs, s.mis, s.S2, s.tmpR, s.prims, n);
		k_children<<<go, 128, 0, st>>>(recs, open_list, nopen, next_list, counters);
		k_owner<<<gn, 256, 0, st>>>(s.owner, recs, n);
		CUB(cudaMemcpyAsync(h, counters, sizeof h, cudaMemcpyDeviceToHost, st));
		CUB(cudaStreamSynchronize(st));
		const uint32_t prev_total = level_first.back() + level_count.back();
		if (h[0] > prev_total) { level_first.push_back(prev_total); level_count.push_back(h[0] - prev_total); }
		k_level_advance<<<1, 1, 0, st>>>(counters);
		h[1] = h[2];
		cur ^= 1;
		if (level_first.size() > BVB_MAX_DEPTH + 2u) return crg_fail(CRGPU_ERR_CUDA, "crgpu_bvh_build: deeper than %u levels", BVB_MAX_DEPTH);
	}
	*nrec_out = h[0];
	return CRGPU_OK;
}

size_t crg_bvh_scratch_bytes(uint32_t n) { Scratch s; return carve(nullptr, n, &s); }

int crg_bvh_build_pairs(const float *bb, const float *ctr, uint32_t n, void *scratch, cudaStream_t st, PairNode *pairs_out, int32_t *prims_out,
					  CrgBuildResult *out) {
	memset(out, 0, sizeof *out);
	if (n == 0u) return CRGPU_OK;
	if (n > 4194304u) return crg_fail(CRGPU_ERR_UNSUPPORTED, "crgpu_bvh_build: %u primitives (limit 4194304 per call)", n);
	Scratch s;
	carve(scratch, n, &s);
	std::vector<uint32_t> level_first, level_count;
	uint32_t nrec = 0u;
	RecStore rs;
	int rc = build_tree(bb, ctr, n, s, st, rs, level_first, level_count, &nrec);
	if (rc) return rc;
	if (nrec > 2u * n - 1u)                                               /* pairs_out, order and bfs_of hold a tree of 2n - 1 nodes */
		return crg_fail(CRGPU_ERR_UNSUPPORTED, "crgpu_bvh_build: the tree of %u primitives needs %u nodes, more than 2n - 1", n, nrec);
	uint32_t info[2] = { 0u, 0u };
	if (nrec > 1u) {
		k_pair_bfs<<<1, 1024, 0, st>>>(rs.recs, s.order, s.bfs_of, s.info);
		const uint32_t internal = (nrec - 1u) / 2u;                   /* a full binary tree */
		k_pairs<<<(internal + 255u) / 256u, 256, 0, st>>>(rs.recs, s.order, s.bfs_of, internal, pairs_out);
		CUB(cudaMemcpyAsync(info, s.info, sizeof info, cudaMemcpyDeviceToHost, st));
	}
	CUB(cudaMemcpyAsync(prims_out, s.prims, (size_t)n * 4u, cudaMemcpyDeviceToDevice, st));
	Rec root;
	CUB(cudaMemcpyAsync(&root, rs.recs, sizeof root, cudaMemcpyDeviceToHost, st));
	CUB(cudaStreamSynchronize(st));
	CUB(cudaGetLastError());
	out->node_count = nrec;
	out->pairs = info[0];
	out->levels = info[1];
	memcpy(out->bounds, root.b, sizeof out->bounds);
	if (nrec == 1u) { out->root_first = root.begin; out->root_count = root.end - root.begin; }
	return CRGPU_OK;
}

extern "C" int crgpu_bvh_build(const float *bboxes, const float *centers, uint32_t n, int device,
								struct crs_bvh_node *nodes_out, uint32_t *node_count_out, int32_t *prims_out) {
	if (!nodes_out || !node_count_out || !prims_out || (n && (!bboxes || !centers))) return crg_fail(CRGPU_ERR_BAD_ARGUMENT, "crgpu_bvh_build: NULL argument");
	*node_count_out = 0u;
	if (n == 0u) return CRGPU_OK;                                           /* bvh.c:251: an empty BVH has no nodes */
	if (n > 4194304u) return crg_fail(CRGPU_ERR_UNSUPPORTED, "crgpu_bvh_build: %u primitives (limit 4194304 per call)", n);
	int ndev = 0;
	int rc = crgpu_device_count(&ndev);
	if (rc) return rc;
	if (device < 0 || device >= ndev) return crg_fail(CRGPU_ERR_BAD_ARGUMENT, "crgpu_bvh_build: device %d out of range (have %d)", device, ndev);
	CUB(cudaSetDevice(device));
	const uint32_t max_rec = 2u * n;
	size_t free_b = 0, total_b = 0;
	CUB(cudaMemGetInfo(&free_b, &total_b));
	const size_t scratch_bytes = crg_bvh_scratch_bytes(n);
	if (scratch_bytes > free_b / 2u) return crg_fail(CRGPU_ERR_NOMEM, "crgpu_bvh_build: %zu bytes of scratch for %u primitives, %zu free", scratch_bytes, n, free_b);
	DevBuf d_bb, d_ctr, d_scratch, d_out;
	CUB(d_bb.alloc((size_t)n * 24u)); CUB(d_ctr.alloc((size_t)n * 12u)); CUB(d_scratch.alloc(scratch_bytes));
	CUB(d_out.alloc((size_t)max_rec * sizeof(crs_bvh_node)));
	Scratch s;
	carve(d_scratch.p, n, &s);
	cudaStream_t st = nullptr;
	CUB(cudaStreamCreateWithFlags(&st, cudaStreamNonBlocking));
	struct StreamGuard { cudaStream_t s; ~StreamGuard() { cudaStreamDestroy(s); } } guard{ st };
	CUB(cudaMemcpyAsync(d_bb.p, bboxes, (size_t)n * 24u, cudaMemcpyHostToDevice, st));
	CUB(cudaMemcpyAsync(d_ctr.p, centers, (size_t)n * 12u, cudaMemcpyHostToDevice, st));
	std::vector<uint32_t> level_first, level_count;
	uint32_t nrec = 0u;
	RecStore rs;
	rc = build_tree(d_bb.as<float>(), d_ctr.as<float>(), n, s, st, rs, level_first, level_count, &nrec);
	if (rc) return rc;
	if (nrec > max_rec - 1u) {                                              /* the caller has room for 2n - 1 nodes */
		*node_count_out = nrec;
		return crg_fail(CRGPU_ERR_UNSUPPORTED, "crgpu_bvh_build: the tree of %u primitives needs %u nodes, more than 2n - 1", n, nrec);
	}
	Rec *recs = rs.recs;
	for (size_t l = level_first.size(); l-- > 0;)
		k_count_internals<<<(level_count[l] + 255u) / 256u, 256, 0, st>>>(recs, level_first[l], level_count[l]);
	for (size_t l = 0; l < level_first.size(); ++l)
		k_assign<<<(level_count[l] + 255u) / 256u, 256, 0, st>>>(recs, level_first[l], level_count[l]);
	k_emit<<<(nrec + 255u) / 256u, 256, 0, st>>>(recs, nrec, d_out.as<crs_bvh_node>());
	CUB(cudaMemcpyAsync(nodes_out, d_out.p, (size_t)nrec * sizeof(crs_bvh_node), cudaMemcpyDeviceToHost, st));
	CUB(cudaMemcpyAsync(prims_out, s.prims, (size_t)n * 4u, cudaMemcpyDeviceToHost, st));
	CUB(cudaStreamSynchronize(st));
	CUB(cudaGetLastError());
	*node_count_out = nrec;
	return CRGPU_OK;
}

/* ---- the top level's inputs for edited instances: instance_bbox of host/loader/cr_sceneload.c ---------------------------------------
 * A mesh starts from its BVH root's bounds as stored (getRootBoundingBox), a sphere from its +-radius box; both go through transformBBox
 * (crl_transform_bbox: every composite the JSON loader builds takes that branch for spheres) and the centre is the box centre (mesh)
 * or A * 0 (sphere).  Plain fp32 operations in the loader's order; -fmad=false keeps them unfused. */
__global__ void k_instance_boxes(const crs_instance *__restrict__ inst, DevInstance *insts, const float *__restrict__ bvh_root, uint32_t n,
								 float *bb, float *ctr, float *offs) {
	const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
	if (i >= n) return;
	DevInstance &d = insts[i];
	if (inst) for (int k = 0; k < 12; ++k) { d.A[k] = inst[i].A[k]; d.Ainv[k] = inst[i].Ainv[k]; }
	const float *m = d.A;                                                     /* rows 0-2 of the row-major 4x4: m[4 * row + col] */
	float mn[3], mx[3];
	if (d.kind == CRS_INST_MESH) {
		const float *b = bvh_root + 6 * (size_t)d.bvh;
		for (int k = 0; k < 3; ++k) { mn[k] = b[2 * k]; mx[k] = b[2 * k + 1]; }
	} else {
		for (int k = 0; k < 3; ++k) { mn[k] = -d.radius; mx[k] = d.radius; }
	}
	float c[3], h[3], lo[3], hi[3];
	for (int k = 0; k < 3; ++k) { c[k] = (mn[k] + mx[k]) * 0.5f; h[k] = (mx[k] - mn[k]) * 0.5f; }
	for (int r = 0; r < 3; ++r) {                                             /* crl_vector / crl_point with |A| in the 3x3 part */
		const float a0 = fabsf(m[4 * r]), a1 = fabsf(m[4 * r + 1]), a2 = fabsf(m[4 * r + 2]);
		const float hr = a0 * h[0] + a1 * h[1] + a2 * h[2];
		const float cr = a0 * c[0] + a1 * c[1] + a2 * c[2] + m[4 * r + 3];
		lo[r] = cr - hr; hi[r] = cr + hr;
	}
	float cen[3];
	for (int r = 0; r < 3; ++r)
		cen[r] = d.kind == CRS_INST_MESH ? (hi[r] + lo[r]) * 0.5f : m[4 * r] * 0.0f + m[4 * r + 1] * 0.0f + m[4 * r + 2] * 0.0f + m[4 * r + 3];
	for (int k = 0; k < 3; ++k) { bb[6 * (size_t)i + k] = lo[k]; bb[6 * (size_t)i + 3 + k] = hi[k]; ctr[3 * (size_t)i + k] = cen[k]; }
	const float ex = hi[0] - lo[0], ey = hi[1] - lo[1], ez = hi[2] - lo[2];
	offs[i] = 0.0001f * sqrtf(ex * ex + ey * ey + ez * ez);                  /* bbox.h:44-46 */
}
/* the reference stores the offset in the object while it builds the top level, so the last instance of an object sets it for all */
__global__ void k_instance_offsets(DevInstance *insts, const uint32_t *__restrict__ last, const float *__restrict__ offs, uint32_t n) {
	const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
	if (i < n) insts[i].ray_offset = offs[last[i]];
}

void crg_launch_instance_boxes(const crs_instance *inst, DevInstance *insts, const float *bvh_root, const uint32_t *last, uint32_t n,
							   float *bb, float *ctr, float *offs, cudaStream_t st) {
	if (n == 0u) return;
	k_instance_boxes<<<(n + 255u) / 256u, 256, 0, st>>>(inst, insts, bvh_root, n, bb, ctr, offs);
	k_instance_offsets<<<(n + 255u) / 256u, 256, 0, st>>>(insts, last, offs, n);
}

/* the edit's item records, from the committed instances' new state and the committed mesh BVH records (a mesh edit moves the pair
 * nodes of the meshes it rebuilds, and may change their node counts and staged prefixes, so those records are written first) */
__global__ void k_top_items(const int32_t *__restrict__ prims, const DevInstance *__restrict__ insts, const DevBvh *__restrict__ bvhs, uint32_t n,
                            DevTopItem *__restrict__ items) {
	const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
	if (i < n) items[i] = crg_top_item(insts[prims[i]], bvhs, (uint32_t)prims[i]);
}
void crg_launch_top_items(const int32_t *prims, const DevInstance *insts, const DevBvh *bvhs, uint32_t n, DevTopItem *items, cudaStream_t st) {
	if (n) k_top_items<<<(n + 255u) / 256u, 256, 0, st>>>(prims, insts, bvhs, n, items);
}

/* ---- a mesh edit's bottom level: poly_bbox, then the records crgpu_prepare packs, in the new leaf order ---------------------------
 * Plain fp32 operations in the loader's / crgpu_prepare's order; -fmad=false keeps the products unfused. */
__global__ void k_poly_boxes(const crs_poly *__restrict__ polys, const float *__restrict__ verts, uint32_t vbase, uint32_t n, float *bb, float *ctr) {
	const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
	if (i >= n) return;
	const crs_poly &p = polys[i];
	const float *v0 = verts + 3 * (size_t)((uint32_t)p.v[0] - vbase), *v1 = verts + 3 * (size_t)((uint32_t)p.v[1] - vbase),
	            *v2 = verts + 3 * (size_t)((uint32_t)p.v[2] - vbase);
	for (int k = 0; k < 3; ++k) {
		bb[6 * (size_t)i + k] = MACRO_MIN(v0[k], MACRO_MIN(v1[k], v2[k]));
		bb[6 * (size_t)i + 3 + k] = MACRO_MAX(v0[k], MACRO_MAX(v1[k], v2[k]));
		ctr[3 * (size_t)i + k] = ((v0[k] + v1[k]) + v2[k]) * (1.0f / 3.0f);
	}
}
void crg_launch_poly_boxes(const crs_poly *polys, const float *verts, uint32_t vbase, uint32_t n, float *bb, float *ctr, cudaStream_t st) {
	if (n) k_poly_boxes<<<(n + 255u) / 256u, 256, 0, st>>>(polys, verts, vbase, n, bb, ctr);
}

__device__ __forceinline__ void cross_unfused(const float *a, const float *b, float *out) {            /* poly.c:22 */
	out[0] = a[1] * b[2] - a[2] * b[1]; out[1] = a[2] * b[0] - a[0] * b[2]; out[2] = a[0] * b[1] - a[1] * b[0];
}
__device__ __forceinline__ void edges(const CrgMeshRepack &m, const crs_poly &p, float *v0, float *e1, float *e2) {   /* poly.c:20-21 */
	const float *a = m.verts + 3 * (size_t)((uint32_t)p.v[0] - m.vbase), *b = m.verts + 3 * (size_t)((uint32_t)p.v[1] - m.vbase),
	            *c = m.verts + 3 * (size_t)((uint32_t)p.v[2] - m.vbase);
	for (int k = 0; k < 3; ++k) { v0[k] = a[k]; e1[k] = a[k] - b[k]; e2[k] = c[k] - a[k]; }
}
/* slot i of the mesh: crgpu_prepare step (2) and the shading key */
__global__ void k_mesh_slots(const CrgMeshRepack m, const int32_t *__restrict__ prims, PackedTri *tris, uint32_t *slot_poly, uint8_t *keys) {
	const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
	if (i >= m.n) return;
	const uint32_t local = (uint32_t)prims[i];
	const crs_poly &p = m.polys[local];
	PackedTri t;
	edges(m, p, t.v0, t.e1, t.e2);
	cross_unfused(t.e1, t.e2, t.n);
	tris[i] = t;
	slot_poly[i] = m.poly_offset + local;
	const uint32_t material = m.material_offset + p.material;
	keys[i] = (uint8_t)(material + 1u < 255u ? material + 1u : 255u);
}
/* poly j of the mesh: crgpu_prepare step (3) */
__global__ void k_mesh_spolys(const CrgMeshRepack m, ShadePoly *spolys) {
	const uint32_t j = blockIdx.x * blockDim.x + threadIdx.x;
	if (j >= m.n) return;
	const crs_poly &p = m.polys[j];
	ShadePoly sp;
	memset(&sp, 0, sizeof sp);
	const bool has_n = p.has_normals != 0;
	if (has_n) {
		float *dst[3] = { sp.n0, sp.n1, sp.n2 };
		for (int v = 0; v < 3; ++v)
			for (int k = 0; k < 3; ++k) dst[v][k] = m.normals[3 * (size_t)((uint32_t)p.n[v] - m.nbase) + k];
	} else {                                                                  /* geometric normal e1 x e2 (poly.c:22,46) */
		float v0[3], e1[3], e2[3];
		edges(m, p, v0, e1, e2);
		cross_unfused(e1, e2, sp.n0);
	}
	const bool has_uv = m.texcoord_count != 0u && p.t[0] != -1;                 /* instance.c:151-153 */
	if (has_uv) {
		float *dst[3] = { sp.t0, sp.t1, sp.t2 };
		for (int v = 0; v < 3; ++v)
			for (int k = 0; k < 2; ++k) dst[v][k] = m.uvs[2 * (size_t)((uint32_t)p.t[v] - m.tbase) + k];
	}
	sp.material = m.material_offset + p.material;
	sp.flags = (has_n ? 1u : 0u) | (has_uv ? 2u : 0u);
	spolys[j] = sp;
}
void crg_launch_mesh_repack(const CrgMeshRepack &m, const int32_t *prims, PackedTri *tris, uint32_t *slot_poly, uint8_t *keys, ShadePoly *spolys,
                            cudaStream_t st) {
	if (!m.n) return;
	k_mesh_slots<<<(m.n + 255u) / 256u, 256, 0, st>>>(m, prims, tris, slot_poly, keys);
	k_mesh_spolys<<<(m.n + 255u) / 256u, 256, 0, st>>>(m, spolys);
}
