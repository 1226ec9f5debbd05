/*
 * crgpu_shade.cu — K3 (shade + compaction), K5 (accumulate), sRGB8 conversion and the known-answer
 * kernel: see crgpu_wave.cuh.  The node interpreter and the fp64 libm stand-ins are real function
 * calls (__noinline__), so the scene descriptor is read through a pointer to its device copy.
 */
#include "crgpu_wave.cuh"
#include "crgpu_shade.cuh"
#include <cstdlib>

/* ---- K4: counting sort of the live rays by shading bucket --------------------------------------------------------------------
 * K2 left the bucket sizes in wb.hist[0..255].  Every block derives the same exclusive prefix, then ranks
 * its rays inside the block with shared-memory atomics and reserves one contiguous range per non-empty bucket
 * with ONE global atomicAdd (cursor = wb.hist[256+k]).  Output: perm[bucket_base + rank] = live index.
 * Order inside a bucket is arbitrary; results do not depend on it (every path carries its own RNG + id). */
#define CRG_BUCKET_ITEMS 8
/* DIR = false: K4 (keys = hitKey, sizes hist[0..255], cursors hist[256..511], output perm).
 * DIR = true:  K4b, the same counting sort over the NEXT bounce's rays by direction bin (keys = dirKey written by K3, sizes
 *              hist[512..767], cursors hist[768..1023], output perm2): K2 hands rays to its lanes in perm2 order, so the 32 rays
 *              of a warp point into the same octant and walk the BVH in the same child order — fewer divergent steps. */
template <bool DIR>
__global__ void __launch_bounds__(256) k_bucket(WaveBuffers wb, int cur, int box_slot, const uint8_t *__restrict__ order, int nflat) {
	__shared__ unsigned s_base[256], s_cnt[256], s_off[256];
	__shared__ unsigned char s_ord[256];
	const unsigned n = wb.counts[cur];
	const unsigned t = threadIdx.x;
	if (DIR && box_slot >= 0 && blockIdx.x == 0u && t < 6u) {   /* K3 is done with this depth's bounds: they key the next batch */
		unsigned *b = wb.box + 12 * box_slot;
		b[6 + t] = b[t];
		b[t] = 0u;
	}
	unsigned *__restrict__ sizes = wb.hist + (DIR ? 512 : 0);
	unsigned *__restrict__ cursors = wb.hist + (DIR ? 768 : 256);
	const unsigned char *__restrict__ keys = DIR ? wb.dirKey : wb.hitKey;
	unsigned *__restrict__ out = DIR ? wb.perm2 : wb.perm;
	s_cnt[t] = sizes[t];
	s_ord[t] = order ? order[t] : (unsigned char)t;
	__syncthreads();
	if (t == 0u) {
		unsigned acc = 0u, flat_end = 0u;
		for (int r = 0; r < 256; ++r) {
			if (r == nflat + 1) flat_end = acc;
			const unsigned k = s_ord[r];
			s_base[k] = acc;
			acc += s_cnt[k];
		}
		/* perm[0 .. counts[4]) are the misses (bucket 0 is always first), perm[counts[4] .. counts[5]) the hits on flat materials */
		if (!DIR && blockIdx.x == 0u) { wb.counts[4] = s_cnt[0]; wb.counts[5] = flat_end; }
	}
	__syncthreads();
	const unsigned chunk = 256u * CRG_BUCKET_ITEMS;
	for (unsigned c0 = blockIdx.x * chunk; c0 < n; c0 += gridDim.x * chunk) {
		s_cnt[t] = 0u;
		__syncthreads();
		unsigned key[CRG_BUCKET_ITEMS], rank[CRG_BUCKET_ITEMS];
#pragma unroll
		for (int k = 0; k < CRG_BUCKET_ITEMS; ++k) {
			const unsigned i = c0 + (unsigned)k * 256u + t;
			key[k] = 0xffffffffu;
			if (i < n) { key[k] = keys[i]; rank[k] = atomicAdd(&s_cnt[key[k]], 1u); }
		}
		__syncthreads();
		s_off[t] = s_cnt[t] ? atomicAdd(&cursors[t], s_cnt[t]) : 0u;
		__syncthreads();
#pragma unroll
		for (int k = 0; k < CRG_BUCKET_ITEMS; ++k) {
			const unsigned i = c0 + (unsigned)k * 256u + t;
			if (key[k] != 0xffffffffu) out[s_base[key[k]] + s_off[key[k]] + rank[k]] = i;
		}
		__syncthreads();
	}
}

/* ---- one bounce of pathTrace's loop body for one path (pathtrace.c:38-57), shared by K3 and the tail kernel -----------------
 * Radiance goes to L[path id].  The reference accumulates into finalColor = (0,0,0) (pathtrace.c:34); the first
 * contribution is therefore written as 0.0f + x (bit-identical, also for x = -0) WITHOUT reading L, and the top bit
 * of the carried id remembers that L holds a value; a path that ends without any contribution writes zeros.  So K1
 * never has to clear L and most paths touch their L record exactly once. */
#define CRG_ID_HAS_L 0x80000000u
CRD void crg_prefetch_l2(const void *p) { asm volatile("prefetch.global.L2 [%0];" ::"l"(p)); }

CRD void cr_add_radiance(float4 *__restrict__ Lbuf, unsigned &id, float r, float g, float b) {
	const unsigned slot = id & ~CRG_ID_HAS_L;
	float4 L = (id & CRG_ID_HAS_L) ? Lbuf[slot] : make_float4(0.0f, 0.0f, 0.0f, 0.0f);
	L.x = L.x + r; L.y = L.y + g; L.z = L.z + b;
	Lbuf[slot] = L;
	id |= CRG_ID_HAS_L;
}
CRD void cr_finish_path(float4 *__restrict__ Lbuf, unsigned id) {
	if (!(id & CRG_ID_HAS_L)) Lbuf[id] = make_float4(0.0f, 0.0f, 0.0f, 0.0f);
}

/* returns true when the path continues with (p_next, d_next) and the updated weight / rng / id */
template <bool X, bool MAYBE_MISS = true, bool FLAT = false>
CRD bool cr_shade_one(const DevScene &sc, float4 *__restrict__ Lbuf, v3 o, v3 d, const Hit &hit, float &wr, float &wg, float &wbl,
					  unsigned &id, uint64_t &rng, int depth, int maxDepth, v3 &p_next, v3 &d_next) {
	if (MAYBE_MISS && hit.inst < 0) {                                                               /* pathtrace.c:39-42 */
		const col4 bg = cr_sample_background<X>(sc, d);
		cr_add_radiance(Lbuf, id, wr * bg.r, wg * bg.g, wbl * bg.b);
		return false;
	}
	Rec rec;
	const int material = cr_reconstruct_hit(sc, o, d, hit, rec, false);
	const DevMaterial mat = sc.materials[material];
	/* pathtrace.c:44.  Without emission (flag 2) the add is x + w*0 == x, skipped, unless w is not finite: then the reference's
	 * sum becomes NaN and so must L (DESIGN.md §2, deviation 4) */
	if ((mat.flags & 2u) || !(isfinite(wr) && isfinite(wg) && isfinite(wbl)))
		cr_add_radiance(Lbuf, id, wr * mat.emission[0], wg * mat.emission[1], wbl * mat.emission[2]);
	if (depth + 1 < maxDepth) {                                                       /* else: the loop ends, the sample is unused */
		BsdfSample s;                                                                 /* pathtrace.c:46-48 */
		if constexpr (FLAT) s = cr_sample_flat(sc, sc.flat[material], rng, rec);
		else s = cr_sample_bsdf<X>(sc, mat.bsdf, rng, rec);
		float probability = 1.0f;
		bool cont = true;
		if (depth >= 4) {                                                             /* pathtrace.c:50-55 */
			probability = CR_MAX(s.color.r, CR_MAX(s.color.g, s.color.b));
			if (cr_draw(rng) > probability) cont = false;
		}
		if (cont) {
			const float inv = cr_div(1.0f, probability);                              /* pathtrace.c:57 */
			wr = (s.color.r * wr) * inv; wg = (s.color.g * wg) * inv; wbl = (s.color.b * wbl) * inv;
			p_next = rec.p; d_next = s.out;
			return true;
		}
	}
	cr_finish_path(Lbuf, id);
	return false;
}

/* order-preserving map of a float to an unsigned (crg_ord(a) < crg_ord(b) iff a < b for non-NaN a, b); never 0 for a finite float */
CRD unsigned crg_ord(float f) { const unsigned u = __float_as_uint(f); return (u & 0x80000000u) ? ~u : (u | 0x80000000u); }
CRD float crg_unord(unsigned e) { return __uint_as_float((e & 0x80000000u) ? (e & 0x7fffffffu) : ~e); }

/* the origin box of dir mode 4: lower corner and 4/extent per axis (0 for a zero or non-finite extent).  Invalid (valid = false)
 * when no origin was reduced into the slot: the first batch of a wave set, or a depth no ray reached. */
struct OriginBox { float lo[3], scale[3]; bool valid; };
CRD OriginBox crg_origin_box(const unsigned *prev) {
	OriginBox b;
	b.valid = true;
	for (int k = 0; k < 3; ++k) {
		if (prev[k] == 0u || prev[3 + k] == 0u) { b.valid = false; b.lo[k] = 0.f; b.scale[k] = 0.f; continue; }
		const float lo = crg_unord(~prev[k]), hi = crg_unord(prev[3 + k]);
		const float e = hi - lo;
		b.lo[k] = lo;
		b.scale[k] = (e > 0.f && e < 3.0e38f) ? 4.0f / e : 0.f;
		if (!(lo <= hi)) b.valid = false;
	}
	return b;
}

/* direction bin of a ray for K4b: sign octant (bvh.c:370-372 picks the near/far planes from exactly these bits), optionally
 * times the major axis or an origin cell.  Any binning is legal: the order rays are traced in never changes a result. */
CRD unsigned cr_dir_bin(const DevScene &sc, const OriginBox &box, v3 o, v3 d, int mode) {
	unsigned key = (__float_as_uint(d.x) >> 31) | ((__float_as_uint(d.y) >> 31) << 1) | ((__float_as_uint(d.z) >> 31) << 2);
	if (mode == 4) {                             /* + 5-bit Morton cell: 4 x 4 x 4 cells of the box, the top 5 of 6 interleaved bits */
		if (!box.valid) return key;
		/* fmaxf(NaN, 0) = 0: a NaN origin or an inf * 0 lands in cell 0 */
		const unsigned cx = (unsigned)fminf(fmaxf((o.x - box.lo[0]) * box.scale[0], 0.0f), 3.0f);
		const unsigned cy = (unsigned)fminf(fmaxf((o.y - box.lo[1]) * box.scale[1], 0.0f), 3.0f);
		const unsigned cz = (unsigned)fminf(fmaxf((o.z - box.lo[2]) * box.scale[2], 0.0f), 3.0f);
		const unsigned m = (cx & 1u) | ((cy & 1u) << 1) | ((cz & 1u) << 2) | ((cx >> 1) << 3) | ((cy >> 1) << 4) | ((cz >> 1) << 5);
		return key | ((m >> 1) << 3);
	}
	if (mode == 2) {
		const float ax = fabsf(d.x), ay = fabsf(d.y), az = fabsf(d.z);
		const unsigned major = (ax >= ay && ax >= az) ? 0u : (ay >= az ? 1u : 2u);
		key |= major << 3;                       /* 0..23 */
	} else if (mode == 3) {                      /* + origin cell in the world box: 4 x 2 x 4 cells -> 256 bins */
		const float fx = (o.x - sc.world_lo[0]) * sc.world_inv[0], fy = (o.y - sc.world_lo[1]) * sc.world_inv[1], fz = (o.z - sc.world_lo[2]) * sc.world_inv[2];
		const unsigned cx = (unsigned)fminf(fmaxf(fx * 4.0f, 0.0f), 3.0f), cy = (unsigned)fminf(fmaxf(fy * 2.0f, 0.0f), 1.0f), cz = (unsigned)fminf(fmaxf(fz * 4.0f, 0.0f), 3.0f);
		key |= (cx << 3) | (cz << 5) | (cy << 7);
	}
	return key;
}

/* ---- K3 (+ compaction) ----------------------------------------------------------------------------------------------
 * PART 0: every ray of the queue.  PART 1 / 3 / 2: the parts of a split launch — 1 = the misses (bucket 0 = perm[0 .. counts[4]):
 * background lookup + radiance, the path always ends, nothing to compact), 3 = the hits on flat materials (perm[counts[4] ..
 * counts[5]): cr_sample_flat, no node interpreter), 2 = the other hits (perm[counts[5] .. n)).  The miss half needs a third of the
 * registers of the hit half, so it runs at twice the occupancy; on hdr.json 40% of all rays are misses and every hit is flat.
 * FLATBG (miss launch only): the scene's background is folded (DevScene::bg) and sampled inline by cr_sample_flat_bg. */
template <int MINB, int PART, bool X, bool FLATBG = false>
__global__ void __launch_bounds__(256, MINB) k_shade(const DevScene *__restrict__ scp, WaveBuffers wb, int cur, int depth, int maxDepth, int dirmode, int prefetch) {
	const DevScene &sc = *scp;
	unsigned n = wb.counts[cur];
	const int nxt = cur ^ 1;
	const unsigned stride = gridDim.x * blockDim.x;
	if (PART == 1) {
		const unsigned n0 = wb.counts[4];
		for (unsigned j = blockIdx.x * blockDim.x + threadIdx.x; j < n0; j += stride) {
			const unsigned i = wb.perm[j];
			const float4 a = crg_half(wb.stA, cur)[i];
			const float4 b = crg_half(wb.stB, cur)[i];
			const uint4 c = crg_half(wb.stC, cur)[i];
			unsigned id = c.y;
			const v3 d = v3make(a.w, b.x, b.y);
			const col4 bg = FLATBG ? cr_sample_flat_bg(sc, sc.bg, d) : cr_sample_background<X>(sc, d);               /* pathtrace.c:39-42 */
			cr_add_radiance(wb.L, id, b.z * bg.r, b.w * bg.g, __uint_as_float(c.x) * bg.b);
		}
		return;
	}
	static_assert(PART != 3 || !X, "the flat launch does not use the node interpreter");
	__shared__ unsigned s_dir[256];                               /* direction-bin sizes of the rays this block writes (blockDim.x == 256) */
	__shared__ unsigned s_box[6];                                 /* dir mode 4: bounds of the origins this block writes (WaveBuffers::box) */
	s_dir[threadIdx.x] = 0u;
	if (threadIdx.x < 6u) s_box[threadIdx.x] = 0u;
	unsigned *box_acc = wb.box + 12 * (depth < CRG_BOX_SLOTS ? depth : CRG_BOX_SLOTS - 1);
	const OriginBox obox = dirmode == 4 ? crg_origin_box(box_acc + 6) : OriginBox{};
	__syncthreads();
	if (PART != 3) {                                              /* the flat launch runs first: the last one resets */
		if (blockIdx.x == 0 && threadIdx.x == 0) wb.counts[2] = 0u;   /* K2's work counter, for the next bounce */
		if (blockIdx.x == 0) { wb.hist[threadIdx.x] = 0u; wb.hist[256 + threadIdx.x] = 0u; }   /* K2/K4 histogram + cursors (blockDim.x == 256) */
	}
	const unsigned lane = threadIdx.x & 31u;
	/* whole warps iterate together so the ballot below is convergent; this launch walks perm[first .. n) */
	const unsigned first = PART == 2 ? wb.counts[5] : (PART == 3 ? wb.counts[4] : 0u);
	if (PART == 3) n = wb.counts[5];
	const unsigned nround = first + ((n - first + 31u) & ~31u);
	/* perm is read two iterations ahead and the records it points to one iteration ahead (crg_prefetch_l2): the five 16-B gathers
	 * through perm are the DRAM-latency loads of this loop (the scene itself is L2-resident), so they are L2 hits when needed */
	unsigned j0 = first + blockIdx.x * blockDim.x + threadIdx.x;
	unsigned i_cur = (prefetch && j0 < n) ? wb.perm[j0] : 0u, i_nxt = (prefetch && j0 + stride < n) ? wb.perm[j0 + stride] : 0u;
	for (unsigned j = j0; j < nround; j += stride) {
		const unsigned i_n2 = (prefetch && j + 2u * stride < n && j + 2u * stride > j) ? wb.perm[j + 2u * stride] : 0u;
		bool alive = false;
		v3 p_next = v3make(0, 0, 0), d_next = v3make(0, 0, 0);
		float wr = 0.f, wg = 0.f, wbl = 0.f;
		unsigned id = 0u;
		uint64_t rng = 0ull;
		if (j < n) {
			const unsigned i = prefetch ? i_cur : wb.perm[j];     /* bucket order: a warp shades one material */
			if (prefetch && j + stride < n) {
				crg_prefetch_l2(&crg_half(wb.stA, cur)[i_nxt]); crg_prefetch_l2(&crg_half(wb.stB, cur)[i_nxt]); crg_prefetch_l2(&crg_half(wb.stC, cur)[i_nxt]);
				crg_prefetch_l2(&wb.hit[i_nxt]); crg_prefetch_l2(&wb.hitInst[i_nxt]);
			}
			const float4 a = crg_half(wb.stA, cur)[i];
			const float4 b = crg_half(wb.stB, cur)[i];
			const uint4 c = crg_half(wb.stC, cur)[i];
			const float4 hq = wb.hit[i];
			Hit hit;
			hit.t = hq.x; hit.u = hq.y; hit.v = hq.z; hit.prim = __float_as_uint(hq.w);
			hit.inst = wb.hitInst[i];
			wr = b.z; wg = b.w; wbl = __uint_as_float(c.x);
			id = c.y;
			rng = (uint64_t)c.z | ((uint64_t)c.w << 32);
			alive = cr_shade_one<X, PART == 0, PART == 3>(sc, wb.L, v3make(a.x, a.y, a.z), v3make(a.w, b.x, b.y), hit, wr, wg, wbl, id, rng, depth, maxDepth, p_next, d_next);
		}
		/* order-preserving warp compaction, one atomic per warp */
		const unsigned mask = __ballot_sync(0xffffffffu, alive);
		if (mask) {
			unsigned base = 0u;
			if (lane == 0u) base = atomicAdd(&wb.counts[nxt], (unsigned)__popc(mask));
			base = __shfl_sync(0xffffffffu, base, 0);
			if (alive) {
				const unsigned k = base + (unsigned)__popc(mask & ((1u << lane) - 1u));
				crg_half(wb.stA, nxt)[k] = make_float4(p_next.x, p_next.y, p_next.z, d_next.x);
				crg_half(wb.stB, nxt)[k] = make_float4(d_next.y, d_next.z, wr, wg);
				crg_half(wb.stC, nxt)[k] = make_uint4(__float_as_uint(wbl), id, (unsigned)(rng & 0xffffffffull), (unsigned)(rng >> 32));
				if (dirmode) {
					const unsigned key = cr_dir_bin(sc, obox, p_next, d_next, dirmode);
					wb.dirKey[k] = (unsigned char)key;
					atomicAdd(&s_dir[key], 1u);
				}
			}
			if (dirmode == 4) {              /* warp-convergent (mask is uniform): min / max of the finite origins written */
				const bool fin = alive && isfinite(p_next.x) && isfinite(p_next.y) && isfinite(p_next.z);
				const float pc[3] = { p_next.x, p_next.y, p_next.z };
#pragma unroll
				for (int c = 0; c < 3; ++c) {
					const unsigned lo = __reduce_max_sync(0xffffffffu, fin ? ~crg_ord(pc[c]) : 0u);
					const unsigned hi = __reduce_max_sync(0xffffffffu, fin ? crg_ord(pc[c]) : 0u);
					if (lane == 0u && hi) { atomicMax(&s_box[c], lo); atomicMax(&s_box[3 + c], hi); }
				}
			}
		}
		i_cur = i_nxt; i_nxt = i_n2;
	}
	if (dirmode) {
		__syncthreads();
		if (s_dir[threadIdx.x]) atomicAdd(&wb.hist[512 + threadIdx.x], s_dir[threadIdx.x]);
		if (dirmode == 4 && threadIdx.x < 6u && s_box[threadIdx.x]) atomicMax(&box_acc[threadIdx.x], s_box[threadIdx.x]);
	}
}

/* ---- tail kernel: when only a handful of paths is left, finish them in ONE launch -------------------------------------------
 * Late bounces hold few rays (hdr.json: <0.1% of the batch after 10 bounces; refraction.json keeps a trickle alive for
 * hundreds of bounces), but every bounce still costs three launches and lasts as long as its slowest ray (~0.2 ms).
 * From bounce CRG_TAIL_FROM on, this kernel is launched before K2: if at most CRG_TAIL_MAX rays are left it runs each
 * remaining path to completion (trace + shade in a per-thread loop — the same device functions, the same draws) and
 * zeroes the live count, so the K2/K4/K3 launches that follow find nothing to do. */
#define CRG_TAIL_MAX 16384u

template <bool X>
__global__ void __launch_bounds__(128) k_tail(const DevScene *__restrict__ scp, WaveBuffers wb, int cur, int depth0, int maxDepth) {
	const DevScene &sc = *scp;
	const unsigned n = wb.counts[cur];
	if (n == 0u || n > CRG_TAIL_MAX) return;
	for (unsigned i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
		const float4 a = crg_half(wb.stA, cur)[i];
		const float4 b = crg_half(wb.stB, cur)[i];
		const uint4 c = crg_half(wb.stC, cur)[i];
		v3 o = v3make(a.x, a.y, a.z), d = v3make(a.w, b.x, b.y);
		float wr = b.z, wg = b.w, wbl = __uint_as_float(c.x);
		unsigned id = c.y;
		uint64_t rng = (uint64_t)c.z | ((uint64_t)c.w << 32);
		unsigned long long rays = 0ull;
		for (int depth = depth0; depth < maxDepth; ++depth) {
			const Hit hit = cr_closest_hit<false>(sc, o, d, nullptr);
			++rays;
			v3 p_next, d_next;
			if (!cr_shade_one<X>(sc, wb.L, o, d, hit, wr, wg, wbl, id, rng, depth, maxDepth, p_next, d_next)) break;
			o = p_next; d = d_next;
		}
		atomicAdd(&wb.stats[0], rays);
	}
	/* the last block to finish clears the queue (every block has read n by then) */
	__shared__ unsigned s_last;
	__syncthreads();
	if (threadIdx.x == 0) { __threadfence(); s_last = atomicAdd(&wb.counts[3], 1u) == gridDim.x - 1u; }
	__syncthreads();
	if (s_last && threadIdx.x == 0) { wb.counts[cur] = 0u; wb.counts[cur ^ 1] = 0u; wb.counts[3] = 0u; }
}

/* ---- K5 ------------------------------------------------------------------------------------------------------------------
 * ARMED (a stoppable scene): the batch is added only if its gates did not abandon it and the running average has reached exactly
 * its first pass — both written by earlier kernels in stream order, so every block takes the same decision.
 * snap_host (a batch that publishes): one thread reads the snapshot state once and tells the publish step that follows whether to
 * stage the image (gate[3]).  K5s run in pass order with a publish step between, so the state read here is what the previous
 * publish step left.
 * VIEWS (crgpu_render_views): px is a piece pixel of the view-major numbering (ViewDesc) and goes to its view's framebuffer with the
 * same walk and arithmetic.  Armed, a views call stages no snapshot: block 0 clears gate[3] so that its publish steps stay one
 * thread's work, and a request stays pending.
 * ADAPTIVE (crgpu_adaptive_round, never with VIEWS): each pass added to a pixel also goes into its record, in pass order: n + 1 and
 * the Welford update of the mean and M2 of the sample's luminance, fp32 under the library's IEEE flags. */
template <bool ARMED, bool VIEWS, bool ADAPTIVE = false>
__global__ void __launch_bounds__(256) k_accumulate(float *__restrict__ fb, const float4 *__restrict__ L, TileDesc td,
													 int image_width, int image_height, unsigned *__restrict__ gate, int set,
													 const unsigned *__restrict__ snap_host, ViewDesc vd, AdaptPix *__restrict__ adapt = nullptr) {
	if (ARMED && VIEWS && blockIdx.x == 0 && threadIdx.x == 0) gate[3] = 0u;
	else if (ARMED && snap_host && blockIdx.x == 0 && threadIdx.x == 0) gate[3] = crg_ld_sys(snap_host + 3) == 1u ? 1u : 0u;
	if (ARMED && (gate[1 + set] != 0u || gate[0] != (unsigned)td.pass_begin)) return;
	const unsigned tile_pixels = td.npix, npass = (unsigned)td.pass_count, P = td.order.p, Q = td.order.q, h = tile_pixels / Q;
	for (unsigned px = blockIdx.x * blockDim.x + threadIdx.x; px < tile_pixels; px += gridDim.x * blockDim.x) {
		int x, y;
		float *img = fb;
		if (VIEWS) {
			unsigned v, tp;
			crg_view_pixel(vd, px, v, tp);
			crg_pixel_xy(td, tp, x, y);
			if (v) img = vd.fb + (size_t)(v - 1u) * vd.fb_floats;
		} else crg_pixel_xy(td, px, x, y);
		const size_t pi = (size_t)x + (size_t)(image_height - (y + 1)) * (size_t)image_width;
		float *dst = img + pi * 3u;                                                                      /* texture.c:24-28 */
		float r = dst[0], g = dst[1], b = dst[2];
		AdaptPix rec;
		if (ADAPTIVE) rec = adapt[pi];
		/* the pixel's passes in pass order (crg_path_pass_pixel): within a pass group its paths are `step` apart, and the whole groups
		 * start P * tile_pixels apart, so only the first group and a last, shorter one need the map.  With P = 1 this is the
		 * pass-major walk L[pass * tile_pixels + px]; with Q = 4 the quarter-warps of a block read 64 contiguous bytes per pass. */
		const unsigned step = px < Q * h ? Q : tile_pixels - Q * h;
		unsigned c0 = 0u, pc = P <= npass ? P : npass, id = crg_path_id(0u, px, tile_pixels, npass, P, Q);
		while (true) {
			for (unsigned j = 0u; j < pc; ++j) {
				const float4 s = L[id + j * step];
				const int completed = td.pass_begin + (int)(c0 + j) + 1;                      /* renderer.c:288-291 */
				const float k = (float)(completed - 1);
				const float t = cr_div(1.0f, (float)completed);
				r = (r * k + s.x) * t; g = (g * k + s.y) * t; b = (b * k + s.z) * t;
				if (ADAPTIVE) {
					const float lum = (0.2126f * s.x + 0.7152f * s.y) + 0.0722f * s.z;
					++rec.n;
					const float d = lum - rec.mean;
					rec.mean = rec.mean + cr_div(d, (float)(rec.n & ~CRG_ADAPT_DONE));
					rec.m2 = rec.m2 + d * (lum - rec.mean);
				}
			}
			c0 += pc;
			if (c0 >= npass) break;
			if (npass - c0 >= P) id += P * tile_pixels;                                     /* the next group is whole */
			else { pc = npass - c0; id = crg_path_id(c0, px, tile_pixels, npass, P, Q); }
		}
		dst[0] = r; dst[1] = g; dst[2] = b;
		if (ADAPTIVE) adapt[pi] = rec;
	}
}

/* ---- adaptive rounds: the convergence test and the active list ----------------------------------------------------------------- */
/* a test point: min_passes + j round_passes below pass_end */
__device__ __forceinline__ bool crg_adapt_test_point(unsigned k, const AdaptParams &a) {
	return k >= a.min_passes && k < a.pass_end && (k - a.min_passes) % a.round_passes == 0u;
}
/* the pixel's record after the test at its count; returns whether it was tested */
__device__ __forceinline__ bool crg_adapt_test(AdaptPix &p, const AdaptParams &a) {
	const unsigned n = p.n & ~CRG_ADAPT_DONE;
	if ((p.n & CRG_ADAPT_DONE) || !crg_adapt_test_point(n, a)) return false;
	const float fn = (float)n;
	p.err = cr_div(__fsqrt_rn(cr_div(cr_div(p.m2, (float)(n - 1u)), fn)), p.mean > a.floor ? p.mean : a.floor);
	if (p.err < a.threshold) p.n |= CRG_ADAPT_DONE;                  /* a NaN error never stops a pixel */
	return true;
}
__device__ __forceinline__ size_t crg_adapt_index(uint32_t xy, int W, int H) {
	return (size_t)(xy & 0xffffu) + (size_t)(H - 1 - (int)(xy >> 16)) * (size_t)W;
}

__global__ void k_adapt_reset(AdaptPix *recs, size_t n) {
	for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x)
		recs[i] = AdaptPix{ 0u, 0.f, 0.f, __int_as_float(0x7f800000) };
}

/* the warps walk the list warp-uniformly, so each warp reduces its min and max before one atomic each */
__global__ void __launch_bounds__(256) k_adapt_select(const uint32_t *__restrict__ pixels, unsigned npix, const AdaptPix *__restrict__ recs,
                                                      int W, int H, AdaptParams a, unsigned long long *__restrict__ flags, unsigned *mm) {
	const unsigned lane = threadIdx.x & 31u, stride = gridDim.x * blockDim.x;
	for (unsigned w0 = blockIdx.x * blockDim.x + (threadIdx.x & ~31u); w0 < npix; w0 += stride) {
		const unsigned i = w0 + lane;
		unsigned lo = 0u, hi = 0u;
		if (i < npix) {
			AdaptPix p = recs[crg_adapt_index(pixels[i], W, H)];
			crg_adapt_test(p, a);
			const unsigned n = p.n & ~CRG_ADAPT_DONE;
			const bool act = !(p.n & CRG_ADAPT_DONE) && n < a.pass_end;
			flags[i] = act ? 1ull : 0ull;
			if (act) { lo = ~n; hi = n; }
		}
		lo = __reduce_max_sync(0xffffffffu, lo);
		hi = __reduce_max_sync(0xffffffffu, hi);
		if (lane == 0u && lo) { atomicMax(mm, lo); atomicMax(mm + 1, hi); }
	}
}

__global__ void __launch_bounds__(256) k_adapt_compact(const uint32_t *__restrict__ pixels, unsigned npix, AdaptPix *__restrict__ recs, int W, int H,
                                                       AdaptParams a, const unsigned long long *__restrict__ flags,
                                                       const unsigned long long *__restrict__ incl, uint32_t *__restrict__ active,
                                                       const unsigned *__restrict__ mm, unsigned *host) {
	const unsigned count = (unsigned)incl[npix - 1u], lo = ~mm[0], hi = mm[1];
	const bool go = count == 0u || lo == hi;                           /* else the round is refused and changes nothing */
	for (unsigned i = blockIdx.x * blockDim.x + threadIdx.x; i < npix; i += gridDim.x * blockDim.x) {
		if (i == 0u) { host[0] = count; host[1] = lo; host[2] = hi; }
		if (!go) continue;
		const uint32_t xy = pixels[i];
		const size_t pi = crg_adapt_index(xy, W, H);
		AdaptPix p = recs[pi];
		if (crg_adapt_test(p, a)) recs[pi] = p;
		if (flags[i]) active[incl[i] - 1ull] = xy;
	}
}

/* colorToSRGB + setPixel(char_p): renderer.c:297-300, texture.c:19-21 */
__global__ void k_to_srgb8(const float *__restrict__ fb, uint8_t *__restrict__ out, size_t n) {
	for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) out[i] = cr_to_srgb8(fb[i]);
}

/* ---- known-answer kernel (parity tests): one thread per (x, y, pass) ---------------------------------------------------------- */
struct HitKat {
	int32_t x, y, pixIdx, instIndex, polyIndex;
	float o[3], d[3];
	float distance, uv[2];
	float hitPoint[3], normal[3];
	float emission[3];
	float out[3], color[4];
	float nextDraw;
	float pad[9];
};

__global__ void k_kat(const DevScene *__restrict__ scp, const int32_t *__restrict__ xyp, int count, HitKat *__restrict__ outv) {
	const DevScene &sc = *scp;
	const int i = blockIdx.x * blockDim.x + threadIdx.x;
	if (i >= count) return;
	HitKat k;
	memset(&k, 0, sizeof k);
	const int x = xyp[3 * i], y = xyp[3 * i + 1], pass = xyp[3 * i + 2];
	k.x = x; k.y = y; k.pixIdx = y * (int)sc.image_width + x;
	uint64_t rng = cr_rng_init((uint32_t)k.pixIdx, (uint32_t)pass, sc.sample_count);
	v3 o, d;
	cr_camera_ray(sc.cam, x, y, rng, o, d);
	k.o[0] = o.x; k.o[1] = o.y; k.o[2] = o.z; k.d[0] = d.x; k.d[1] = d.y; k.d[2] = d.z;
	const Hit hit = cr_closest_hit<false>(sc, o, d, nullptr);
	k.instIndex = hit.inst;
	BsdfSample s;
	if (hit.inst < 0) {
		k.polyIndex = -1;
		s.out = v3make(0.f, 0.f, 0.f);
		s.color = cr_sample_background<true>(sc, d);
	} else {
		Rec rec;
		const int material = cr_reconstruct_hit(sc, o, d, hit, rec, true);
		const DevInstance *inst = sc.instances + hit.inst;
		k.polyIndex = inst->kind == CRS_INST_MESH ? (int)sc.slot_poly[hit.prim] : -1;
		k.distance = hit.t; k.uv[0] = rec.uv.x; k.uv[1] = rec.uv.y;
		k.hitPoint[0] = rec.p.x; k.hitPoint[1] = rec.p.y; k.hitPoint[2] = rec.p.z;
		k.normal[0] = rec.n.x; k.normal[1] = rec.n.y; k.normal[2] = rec.n.z;
		const DevMaterial mat = sc.materials[material];
		k.emission[0] = mat.emission[0]; k.emission[1] = mat.emission[1]; k.emission[2] = mat.emission[2];
		s = cr_sample_bsdf<true>(sc, mat.bsdf, rng, rec);
	}
	k.out[0] = s.out.x; k.out[1] = s.out.y; k.out[2] = s.out.z;
	k.color[0] = s.color.r; k.color[1] = s.color.g; k.color[2] = s.color.b; k.color[3] = s.color.a;
	k.nextDraw = cr_draw(rng);
	outv[i] = k;
}

void crg_launch_bucket(const WaveBuffers &wb, int cur, int grid, const uint8_t *order, int nflat, cudaStream_t st) {
	k_bucket<false><<<grid, 256, 0, st>>>(wb, cur, -1, order, nflat);
}
/* X (the last template argument): the scene contains node kinds only the complete interpreter knows (DevScene::has_xnodes, set at
 * upload) — every other scene runs the kernels in which that interpreter is not even linked */
void crg_launch_tail(const DevScene *dsc, const WaveBuffers &wb, int cur, int depth, int maxDepth, bool xnodes, cudaStream_t st) {
	if (xnodes) k_tail<true><<<128, 128, 0, st>>>(dsc, wb, cur, depth, maxDepth);
	else k_tail<false><<<128, 128, 0, st>>>(dsc, wb, cur, depth, maxDepth);
}
/* CRGPU_SHADE_MINB = 2|3|4 (blocks per SM of the hit/all kernel: 128 / 80 / 64 registers), CRGPU_SHADE_SPLIT = 0|1 (separate
 * miss kernel at 4 blocks per SM), CRGPU_SHADE_PREFETCH = 0|1 — read once; the defaults are what measured best.  On an H100 80GB HBM3
 * at a 400 W limit (hdr.json, 1080p, 1000 spp) the shading step takes 720 ms per frame with the hit kernel at 2 blocks per SM, 883 ms at 3 and 1068 ms at 4.
 * ptxas reports 784 B of spill stores for the hit kernel at 80 registers and 124 B at 128.
 * CRGPU_SHADE_GENERIC_ONLY = 0|1 (1: no flat launch), CRGPU_SHADE_FLAT_MINB = 2|3|4: the flat hit kernel needs no call and no spill at
 * 80 registers, and on an H100 80GB HBM3 at 700 W its shading step takes 481 ms per frame at 3 blocks per SM, 499 ms at 2, 502 ms at 4
 * (616 ms with every hit through the interpreter). */
const ShadeKnobs &crg_shade_knobs_env(void) {
	static const ShadeKnobs kn = [] {
		ShadeKnobs k;
		const char *e = getenv("CRGPU_SHADE_MINB");
		const int v = e ? atoi(e) : 2;
		k.minb = v >= 2 && v <= 4 ? v : 2;
		e = getenv("CRGPU_SHADE_SPLIT");
		k.split = e ? atoi(e) : 1;
		e = getenv("CRGPU_SHADE_PREFETCH");
		k.prefetch = e ? atoi(e) : 0;
		e = getenv("CRGPU_SHADE_GENERIC_ONLY");
		k.generic_only = e ? atoi(e) != 0 : 0;
		e = getenv("CRGPU_SHADE_FLAT_MINB");
		const int f = e ? atoi(e) : 3;
		k.flat_minb = f >= 2 && f <= 4 ? f : 3;
		return k;
	}();
	return kn;
}
template <bool X>
static int launch_shade(const DevScene *dsc, const WaveBuffers &wb, int cur, int depth, int maxDepth, int dirmode, int grid, const ShadeKnobs &kn,
                        bool flat_bg, cudaStream_t st, cudaEvent_t *ev) {
	const int minb = kn.minb, split = kn.split, prefetch = kn.prefetch;
	if (split) {
		if (flat_bg) k_shade<4, 1, X, true><<<grid, 256, 0, st>>>(dsc, wb, cur, depth, maxDepth, dirmode, prefetch);
		else k_shade<4, 1, X><<<grid, 256, 0, st>>>(dsc, wb, cur, depth, maxDepth, dirmode, prefetch);
		if (ev) cudaEventRecord(ev[0], st);
		if (!kn.generic_only) {                                      /* perm[counts[4] .. counts[5]): the flat materials */
			if (kn.flat_minb == 3) k_shade<3, 3, false><<<grid, 256, 0, st>>>(dsc, wb, cur, depth, maxDepth, dirmode, prefetch);
			else if (kn.flat_minb == 4) k_shade<4, 3, false><<<grid, 256, 0, st>>>(dsc, wb, cur, depth, maxDepth, dirmode, prefetch);
			else k_shade<2, 3, false><<<grid, 256, 0, st>>>(dsc, wb, cur, depth, maxDepth, dirmode, prefetch);
		}
		if (ev) cudaEventRecord(ev[1], st);
		if (minb == 3) k_shade<3, 2, X><<<grid, 256, 0, st>>>(dsc, wb, cur, depth, maxDepth, dirmode, prefetch);
		else if (minb == 4) k_shade<4, 2, X><<<grid, 256, 0, st>>>(dsc, wb, cur, depth, maxDepth, dirmode, prefetch);
		else k_shade<2, 2, X><<<grid, 256, 0, st>>>(dsc, wb, cur, depth, maxDepth, dirmode, prefetch);
		if (ev) cudaEventRecord(ev[2], st);
		return kn.generic_only ? 2 : 3;
	}
	if (minb == 3) k_shade<3, 0, X><<<grid, 256, 0, st>>>(dsc, wb, cur, depth, maxDepth, dirmode, prefetch);
	else if (minb == 4) k_shade<4, 0, X><<<grid, 256, 0, st>>>(dsc, wb, cur, depth, maxDepth, dirmode, prefetch);
	else k_shade<2, 0, X><<<grid, 256, 0, st>>>(dsc, wb, cur, depth, maxDepth, dirmode, prefetch);
	if (ev) for (int k = 0; k < 3; ++k) cudaEventRecord(ev[k], st);   /* one launch: it is all in the "miss" share */
	return 1;
}
int crg_launch_shade(const DevScene *dsc, const WaveBuffers &wb, int cur, int depth, int maxDepth, int dirmode, bool xnodes, bool flat_bg, int grid,
                     const ShadeKnobs &kn, cudaStream_t st, cudaEvent_t *ev) {
	if (xnodes) return launch_shade<true>(dsc, wb, cur, depth, maxDepth, dirmode, grid, kn, flat_bg, st, ev);
	return launch_shade<false>(dsc, wb, cur, depth, maxDepth, dirmode, grid, kn, flat_bg, st, ev);
}
void crg_launch_dirsort(const WaveBuffers &wb, int nxt, int box_slot, int grid, cudaStream_t st) {
	k_bucket<true><<<grid, 256, 0, st>>>(wb, nxt, box_slot, nullptr, 0);
}
int crg_dir_mode(void) {
	static const int mode = [] { const char *e = getenv("CRGPU_TRACE_SORT"); const int v = e ? atoi(e) : 0; return v >= 0 && v <= 4 ? v : 0; }();
	return mode;
}
bool crg_shade_flat_order(const ShadeKnobs &kn) { return kn.split && !kn.generic_only; }

/* ---- the libm stand-ins one by one (test entry crgpu_libm_eval; the order of include/crgpu.h CRGPU_LIBM_*) -------------------- */
__global__ void k_libm(int fn, const float *__restrict__ x, const float *__restrict__ y, float *__restrict__ out, unsigned n) {
	for (unsigned i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
		const float a = x[i], b = y[i];
		float r, s, c;
		switch (fn) {
		case 0: r = cr_sinf(a); break;
		case 1: r = cr_cosf(a); break;
		case 2: r = cr_tanf(a); break;
		case 3: r = cr_logf(a); break;
		case 4: r = cr_log10f(a); break;
		case 5: r = cr_atan2f(a, b); break;
		case 6: r = cr_acosf(a); break;
		case 7: r = cr_asinf(a); break;
		case 8: r = cr_powf(a, b); break;
		case 9: r = cr_pow5f(a); break;
		case 10: cr_sincosf(a, &s, &c); r = s; break;
		default: cr_sincosf(a, &s, &c); r = c; break;
		}
		out[i] = r;
	}
}
void crg_launch_libm(int fn, const float *x, const float *y, float *out, unsigned n, cudaStream_t st) {
	k_libm<<<256, 256, 0, st>>>(fn, x, y, out, n);
}
void crg_launch_accumulate(float *fb, const float4 *L, const TileDesc &td, int W, int H, int grid, cudaStream_t st, unsigned *gate, int set,
                           const unsigned *snap_host, const ViewDesc *vd, AdaptPix *adapt) {
	if (adapt) {
		if (gate) k_accumulate<true, false, true><<<grid, 256, 0, st>>>(fb, L, td, W, H, gate, set, snap_host, ViewDesc{}, adapt);
		else k_accumulate<false, false, true><<<grid, 256, 0, st>>>(fb, L, td, W, H, nullptr, 0, nullptr, ViewDesc{}, adapt);
	} else if (vd) {
		if (gate) k_accumulate<true, true><<<grid, 256, 0, st>>>(fb, L, td, W, H, gate, set, nullptr, *vd);
		else k_accumulate<false, true><<<grid, 256, 0, st>>>(fb, L, td, W, H, nullptr, 0, nullptr, *vd);
	} else if (gate) k_accumulate<true, false><<<grid, 256, 0, st>>>(fb, L, td, W, H, gate, set, snap_host, ViewDesc{});
	else k_accumulate<false, false><<<grid, 256, 0, st>>>(fb, L, td, W, H, nullptr, 0, nullptr, ViewDesc{});
}
void crg_launch_adapt_reset(AdaptPix *recs, size_t n, cudaStream_t st) { k_adapt_reset<<<1024, 256, 0, st>>>(recs, n); }
void crg_launch_adapt_select(const uint32_t *pixels, unsigned npix, const AdaptPix *recs, int W, int H, const AdaptParams &a,
                             unsigned long long *flags, unsigned *mm, cudaStream_t st) {
	const unsigned grid = (npix + 255u) / 256u < 4096u ? (npix + 255u) / 256u : 4096u;
	k_adapt_select<<<grid, 256, 0, st>>>(pixels, npix, recs, W, H, a, flags, mm);
}
void crg_launch_adapt_compact(const uint32_t *pixels, unsigned npix, AdaptPix *recs, int W, int H, const AdaptParams &a,
                              const unsigned long long *flags, const unsigned long long *incl, uint32_t *active, const unsigned *mm,
                              unsigned *host, cudaStream_t st) {
	const unsigned grid = (npix + 255u) / 256u < 4096u ? (npix + 255u) / 256u : 4096u;
	k_adapt_compact<<<grid, 256, 0, st>>>(pixels, npix, recs, W, H, a, flags, incl, active, mm, host);
}
void crg_launch_to_srgb8(const float *fb, uint8_t *out, size_t n, int grid, cudaStream_t st) {
	k_to_srgb8<<<grid, 256, 0, st>>>(fb, out, n);
}
void crg_launch_kat(const DevScene *dsc, const int32_t *xyp, int count, void *out, cudaStream_t st) {
	k_kat<<<(count + 63) / 64, 64, 0, st>>>(dsc, xyp, count, static_cast<HitKat *>(out));
}
static_assert(sizeof(HitKat) == 160, "HitKat must match struct hit_kat of oracle/ref_harness.c");
