/*
 * crgpu_trace.cu — K1 (primary-ray generation) and K2 (two-level BVH traversal): see crgpu_wave.cuh.
 * Everything here is force-inlined; the scene descriptor travels as a by-value kernel parameter so
 * its pointers sit in the constant bank.
 */
#include <mutex>
#include "crgpu_wave.cuh"
#include "crgpu_trace.cuh"
#include <cstdlib>

/* ---- pixel list of a tile set: blockIdx.y = tile, the block's threads walk its pixels row by row, or in 8x4 blocks (blocked,
 *      crg_block_xy) (crgpu_render_tiles) ------------------------------------------------------------------------------------------- */
__global__ void __launch_bounds__(256) k_pixel_list(uint32_t *__restrict__ pixels, const int4 *__restrict__ rects, const unsigned *__restrict__ offs, int blocked) {
	const int4 r = rects[blockIdx.y];
	const unsigned w = (unsigned)(r.z - r.x), h = (unsigned)(r.w - r.y), n = w * h;
	uint32_t *out = pixels + offs[blockIdx.y];
	for (unsigned i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
		unsigned x, y;
		if (blocked) crg_block_xy(i, w, h, x, y);
		else { y = i / w; x = i - y * w; }
		out[i] = (uint32_t)(r.x + (int)x) | ((uint32_t)(r.y + (int)y) << 16);
	}
}
void crg_launch_pixel_list(uint32_t *pixels, const int4 *rects, const unsigned *offs, int nrects, int blocked, cudaStream_t st) {
	for (int first = 0; first < nrects; first += 32768) {            /* gridDim.y <= 65535 */
		const int cnt = nrects - first < 32768 ? nrects - first : 32768;
		k_pixel_list<<<dim3(4, (unsigned)cnt), 256, 0, st>>>(pixels, rects + first, offs + first, blocked);
	}
}

/* CRGPU_PATH_ORDER (crg_path_order_of), read once per process; any value outside 0 .. CRG_PATH_ORDERS - 1 selects the default.
 * 6 (16 passes of a 2x1 pixel pair per warp): on hdr.json (1080p, 1000 spp, one H100 80GB HBM3 at 700 W) bench.py measures
 * 4696-4698 Mray/s against 4680-4683 in order 2 and 4534-4578 in order 0's build before the knob (DESIGN §4) */
#define CRG_PATH_ORDER_DEFAULT 6
const PathOrder &crg_path_order(void) {
	static const PathOrder o = [] {
		const char *e = getenv("CRGPU_PATH_ORDER");
		const int v = e ? atoi(e) : CRG_PATH_ORDER_DEFAULT;
		return crg_path_order_of(v >= 0 && v < CRG_PATH_ORDERS ? v : CRG_PATH_ORDER_DEFAULT);
	}();
	return o;
}

/* ---- K1 ------------------------------------------------------------------------------------------------------------
 * VIEWS (crgpu_render_views): px is a piece pixel of the view-major numbering (ViewDesc), and the ray is taken from its view's camera
 * with the same arithmetic; vd is unused otherwise. */
template <bool VIEWS>
__global__ void __launch_bounds__(256) k_generate(DevScene sc, WaveBuffers wb, TileDesc td, ViewDesc vd) {
	const unsigned tile_pixels = td.npix;
	const unsigned n = tile_pixels * (unsigned)td.pass_count;
	for (unsigned id = blockIdx.x * blockDim.x + threadIdx.x; id < n; id += gridDim.x * blockDim.x) {
		unsigned pl, px;
		crg_path_pass_pixel(id, tile_pixels, (unsigned)td.pass_count, td.order.p, td.order.q, pl, px);
		int x, y;
		unsigned v = 0u;
		if (VIEWS) { unsigned tp; crg_view_pixel(vd, px, v, tp); crg_pixel_xy(td, tp, x, y); }
		else crg_pixel_xy(td, px, x, y);
		const uint32_t pixIdx = (uint32_t)(y * (int)sc.image_width + x);                        /* renderer.c:280 */
		uint64_t rng = cr_rng_init(pixIdx, (uint32_t)(td.pass_begin + (int)pl), sc.sample_count);
		v3 o, d;
		if (VIEWS) cr_camera_ray(*(v ? vd.cams + (v - 1u) : vd.cam0), x, y, rng, o, d);
		else cr_camera_ray(sc.cam, x, y, rng, o, d);
		wb.stA[0][id] = make_float4(o.x, o.y, o.z, d.x);
		wb.stB[0][id] = make_float4(d.y, d.z, 1.0f, 1.0f);
		wb.stC[0][id] = make_uint4(__float_as_uint(1.0f), id, (unsigned)(rng & 0xffffffffull), (unsigned)(rng >> 32));
	}
	if (blockIdx.x == 0 && threadIdx.x == 0) { wb.counts[0] = n; wb.counts[1] = 0u; wb.counts[2] = 0u; wb.counts[3] = 0u; }
	if (blockIdx.x == 0) { for (int k = 0; k < 4; ++k) wb.hist[k * 256 + threadIdx.x] = 0u; }   /* blockDim.x == 256 */
}

/* ---- K2: persistent warps with dynamic ray refill ----------------------------------------------------------------------
 * Ray lengths vary a lot (hdr.json: 7 child-pair steps on average, >200 for some), so a warp that takes 32
 * rays and waits for the slowest one idles most lanes (ncu: 7-10 active threads/warp).  Here every warp keeps
 * its 32 traversal state machines in registers and, whenever fewer than CRG_REFILL lanes are busy, pulls new
 * rays for the idle lanes from a global work counter (one ballot + one atomicAdd per refill, indices handed
 * out in lane order so neighbouring lanes still get neighbouring — coherent — rays). */
#define CRG_REFILL 16
#define CRG_NODE_BURST 3
#define CRG_STAGE_MIN_RAYS 65536u
#define CRG_DEFER_DEFAULT 0
/* lanes that must want an instance step before a warp takes one: on hdr.json (1080p, 1000 spp, one H100 80GB HBM3 at 700 W)
 * 4 renders the frame 0.7% faster than 8 and 12 1.4% slower (tools/k2_order_sweep.py, DESIGN §4) */
#define CRG_INST_MIN 4
#define CRG_MAX_STEPS 8000000u   /* > 30x the node count of any scene that fits the 2^23-node address space we support */

template <bool COUNT, int MINB, int DEFER>
__global__ void __launch_bounds__(256, MINB) k_trace(DevScene sc, WaveBuffers wb, int cur, int refill, int burst, int sorted, int inst_min) {
	const unsigned n = wb.counts[cur];
	const unsigned lane = threadIdx.x & 31u;
	const float4 *__restrict__ stA = crg_half(wb.stA, cur);
	const float4 *__restrict__ stB = crg_half(wb.stB, cur);
	TraceCounters tc = { 0u, 0u, 0u, 0u };
	__shared__ unsigned s_hist[256];
	__shared__ CoopScratch s_coop[DEFER == 2 ? 8 : 1];   /* one per warp (blockDim.x == 256) */
	s_hist[threadIdx.x] = 0u;            /* blockDim.x == 256 */
	/* K3 + K4b of the previous bounce are done with the direction-bin counters: clear them for this bounce's K3 */
	if (blockIdx.x == 0) { wb.hist[512 + threadIdx.x] = 0u; wb.hist[768 + threadIdx.x] = 0u; }
	const unsigned *__restrict__ order = sorted ? wb.perm2 : nullptr;     /* rays in direction-bin order (see k_dirsort) */
	__syncthreads();
	/* ---- stage the top-of-tree pair nodes into shared memory: one TMA bulk copy (cp.async.bulk, SASS UBLKCP) per
	 *      block, completion signalled on an mbarrier; skipped for the small tail launches where it cannot pay off */
	__shared__ __align__(8) unsigned long long s_mbar;
	bool staged = false;
	if (sc.stage_pairs && n >= CRG_STAGE_MIN_RAYS) {
		const unsigned bytes = sc.stage_pairs * (unsigned)sizeof(PairNode);
		const unsigned mbar = (unsigned)__cvta_generic_to_shared(&s_mbar);
		const unsigned dst = (unsigned)__cvta_generic_to_shared(crg_stage_smem);
		if (threadIdx.x == 0) {
			asm volatile("mbarrier.init.shared::cta.b64 [%0], 1;" ::"r"(mbar));
			asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
		}
		__syncthreads();
		if (threadIdx.x == 0) {
			asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(mbar), "r"(bytes) : "memory");
			asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
						 ::"r"(dst), "l"(sc.stage_img), "r"(bytes), "r"(mbar) : "memory");
		}
		unsigned ok = 0u;
		while (!ok) {
			asm volatile("{\n\t.reg .pred p;\n\tmbarrier.try_wait.parity.shared::cta.b64 p, [%1], 0;\n\tselp.u32 %0, 1, 0, p;\n\t}"
						 : "=r"(ok) : "r"(mbar) : "memory");
		}
		staged = true;
	}
	uint32_t ovf[CRG_OVF];           /* the traversal stack below its top CRG_SSTACK entries (those are in shared memory) */
	Traversal<COUNT> tr;
	tr.begin(sc, v3make(0.f, 0.f, 0.f), v3make(0.f, 0.f, 1.f), staged);   /* every lane holds a VALID (idle) state from the start */
	bool busy = false;
	bool exhausted = false;          /* warp-uniform: the work counter ran past n */
	unsigned ray = 0u;
	unsigned steps = 0u;             /* safety net: a lane that exceeds CRG_MAX_STEPS is abandoned and flagged */
	while (true) {
		unsigned active = __ballot_sync(0xffffffffu, busy);
		if (!exhausted && __popc(active) < refill) {
			const unsigned idle = ~active;
			const unsigned nidle = (unsigned)__popc(idle);
			unsigned base = 0u;
			if (lane == 0u) base = atomicAdd(&wb.counts[2], nidle);
			base = __shfl_sync(0xffffffffu, base, 0);
			if (base + nidle >= n) exhausted = true;
			const unsigned slot = base + (unsigned)__popc(idle & ((1u << lane) - 1u));
			if (!busy && slot < n) {
				const unsigned i = order ? order[slot] : slot;
				const float4 a = stA[i];
				const float4 b = stB[i];
				ray = i;
				steps = 0u;
				tr.begin(sc, v3make(a.x, a.y, a.z), v3make(a.w, b.x, b.y), staged);
				busy = true;
			}
			active = __ballot_sync(0xffffffffu, busy);
		}
		if (active == 0u) break;         /* nothing in flight and nothing left to fetch */
		/* Phase N: up to CRG_NODE_BURST child-pair steps for every lane that is inside a BVH.  Lanes that reach a
		 * top-level leaf (instance work) or finish wait here, so that the instance / write-back code below runs
		 * for many lanes at once instead of being serialised against node steps in every iteration. */
#pragma unroll 1
		for (int k = 0; k < burst; ++k) {
			const bool wn = busy && tr.wants_node();
			if (!__any_sync(0xffffffffu, wn)) break;
			if (wn) { tr.template node_step<DEFER != 0>(sc, ovf, &tc); ++steps; }
		}
		/* Phase T (DEFER): the triangles of every lane that reached a leaf during the burst, together */
		if (DEFER == 2) cr_coop_leaves<COUNT>(tr, busy && tr.wants_leaf(), sc, s_coop[threadIdx.x >> 5], lane, &tc);   /* dealt over the warp */
		else if (DEFER == 1 && busy && tr.wants_leaf()) tr.leaf_step(sc, &tc);
		/* Phase I: one pending instance (ray transform + sphere test, or entry into a mesh BVH).  ncu (19.8% of K2's
		 * warp instructions ran with fewer than 2 active lanes, almost all of them here): lanes reach a top-level leaf at different
		 * iterations, so running this ~100-instruction block whenever ANY lane wants it means running it for one lane.  Lanes
		 * therefore WAIT here until at least `inst_min` of them want an instance step, or no lane of the warp can take a node step. */
		{
			const bool wi = busy && tr.wants_instance();
			const unsigned mi = __ballot_sync(0xffffffffu, wi);
			if (mi) {
				bool go = (int)__popc(mi) >= inst_min;
				if (!go) go = !__any_sync(0xffffffffu, busy && tr.wants_node());
				if (go && wi) { tr.instance_step(sc, &tc); ++steps; }
			}
		}
		/* Phase W: write back finished rays */
		if (busy && tr.done()) {
			const Hit best = tr.result();
			wb.hit[ray] = make_float4(best.t, best.u, best.v, __uint_as_float(best.prim));
			wb.hitInst[ray] = best.inst;
			unsigned key = 0u;                                   /* shading bucket for K4/K3: one byte load (DevScene::slot_key) */
			if (best.inst >= 0) key = (tr.flags & CRG_TF_SPHERE) ? __ldg(sc.inst_key + best.inst) : __ldg(sc.slot_key + best.prim);
			wb.hitKey[ray] = (unsigned char)key;
			atomicAdd(&s_hist[key], 1u);
			busy = false;
		} else if (busy && steps > CRG_MAX_STEPS) {              /* cannot happen for a finite BVH; never hang the GPU */
			atomicAdd(&wb.stats[7], 1ull);
			wb.hit[ray] = make_float4(CR_FLT_MAX, 0.f, 0.f, 0.f);
			wb.hitInst[ray] = -1;
			wb.hitKey[ray] = 0;
			atomicAdd(&s_hist[0], 1u);
			busy = false;
		}
	}
	__syncthreads();
	if (s_hist[threadIdx.x]) atomicAdd(&wb.hist[threadIdx.x], s_hist[threadIdx.x]);
	if (COUNT) {
		atomicAdd(&wb.stats[1], (unsigned long long)tc.pairs);
		atomicAdd(&wb.stats[2], (unsigned long long)tc.tris);
		atomicAdd(&wb.stats[3], (unsigned long long)tc.spheres);
		atomicAdd(&wb.stats[4], (unsigned long long)tc.insts);
	}
	if (blockIdx.x == 0 && threadIdx.x == 0) {
		atomicAdd(&wb.stats[0], (unsigned long long)n);          /* one ray per getClosestIsect (two streams may run two K2s) */
		wb.counts[cur ^ 1] = 0u;   /* K3 of this bounce appends survivors there */
	}
}

void crg_launch_generate(const DevScene &sc, const WaveBuffers &wb, const TileDesc &td, const ViewDesc *vd, int grid, cudaStream_t st) {
	if (vd) k_generate<true><<<grid, 256, 0, st>>>(sc, wb, td, *vd);
	else k_generate<false><<<grid, 256, 0, st>>>(sc, wb, td, ViewDesc{});
}

/* ---- stop gates of an armed scene (crgpu_wave.cuh): one thread each, but for a publish step that stages a snapshot ------------------
 * The host words are read and written at system scope (crg_ld_sys / crg_st_sys). */
__global__ void k_stop_gate(unsigned *counts, int cur, unsigned *ctl, int set, const unsigned *host, int reset, int check) {
	unsigned ab = reset ? 0u : ctl[1 + set];
	if (!ab && check) ab = crg_ld_sys(host) != 0u ? 1u : 0u;
	ctl[1 + set] = ab;
	if (ab) { counts[cur] = 0u; counts[cur ^ 1] = 0u; counts[3] = 0u; }   /* exactly what k_tail's last block clears */
}
__global__ void k_stop_begin(unsigned *ctl, unsigned *host, int pass_begin) {
	ctl[0] = (unsigned)pass_begin;
	crg_st_sys(host + 1, (unsigned)pass_begin);
	crg_st_sys(host + 2, 1u);
	__threadfence_system();
}
/* Block 0's thread 0 publishes.  A snapshot (ctl[3], decided by K5 from the host state) is the framebuffer as K5 left it: exactly
 * the passes [call's pass_begin, ctl[0]).  The next K5 to write the framebuffer waits for this kernel in stream order, so the image
 * holds no later batch.  The last block to finish stages it: the pass index first, then the state, so that a host that sees
 * "staged" reads the index and image of this step, never one the progress word has not yet reached. */
__global__ void __launch_bounds__(256) k_stop_publish(unsigned *ctl, int set, unsigned *host, int pass_begin, int pass_count,
                                                      unsigned long long paths, unsigned long long *stats, const float *__restrict__ fb,
                                                      uint8_t *__restrict__ snap, size_t n) {
	if (blockIdx.x == 0 && threadIdx.x == 0) {
		if (ctl[1 + set] == 0u && ctl[0] == (unsigned)pass_begin) {       /* the decision K5 took */
			ctl[0] = (unsigned)(pass_begin + pass_count);
			stats[5] += paths;
		}
		crg_st_sys(host + 1, ctl[0]);
		__threadfence_system();
	}
	if (ctl[3] == 0u) return;                                             /* no snapshot requested: the usual one-thread step */
	for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) snap[i] = cr_to_srgb8(fb[i]);
	__threadfence();
	__syncthreads();
	if (threadIdx.x == 0 && atomicAdd(&ctl[4], 1u) == gridDim.x - 1u) {
		ctl[4] = 0u;
		crg_st_sys(host + 4, *(volatile unsigned *)&ctl[0]);            /* block 0 wrote it before its count */
		__threadfence_system();
		crg_st_sys(host + 3, 2u);
		__threadfence_system();
	}
}
__global__ void k_stop_end(const unsigned *ctl, unsigned *host) {
	crg_st_sys(host + 1, ctl[0]);
	__threadfence_system();
	crg_st_sys(host + 2, 0u);
	__threadfence_system();
}
void crg_launch_stop_gate(unsigned *counts, int cur, unsigned *ctl, int set, const unsigned *host, bool reset, bool check, cudaStream_t st) {
	k_stop_gate<<<1, 1, 0, st>>>(counts, cur, ctl, set, host, reset ? 1 : 0, check ? 1 : 0);
}
void crg_launch_stop_begin(unsigned *ctl, unsigned *host, int pass_begin, cudaStream_t st) { k_stop_begin<<<1, 1, 0, st>>>(ctl, host, pass_begin); }
void crg_launch_stop_publish(unsigned *ctl, int set, unsigned *host, int pass_begin, int pass_count, unsigned long long paths,
                             unsigned long long *stats, const float *fb, uint8_t *snap, size_t n, int grid, cudaStream_t st) {
	k_stop_publish<<<grid, 256, 0, st>>>(ctl, set, host, pass_begin, pass_count, paths, stats, fb, snap, n);
}
void crg_launch_stop_end(unsigned *ctl, unsigned *host, cudaStream_t st) { k_stop_end<<<1, 1, 0, st>>>(ctl, host); }
/* K2 is persistent: the grid is exactly the number of blocks the device can keep resident (the occupancy query below also
 * counts the staged nodes' dynamic shared memory, so CRGPU_TRACE_STAGE=1024 gets fewer blocks).  MINB (blocks per SM the compiler
 * must make room for: 2 -> <=128 registers, 3 -> <=80, 4 -> <=64) trades registers for latency-hiding warps.  K2 is bound by
 * latency, and with its cold state and the top of its stack in shared memory it runs at 64 registers with 30 B of spills, so the
 * default is 4 (32 warps per SM): on hdr.json (1080p, 1000 spp, one H100 80GB HBM3 at 400 W) 4 traces the frame in 854 ms, 3 in
 * 901 ms (DESIGN §4).  CRGPU_TRACE_MINB=2|3 selects the others. */
#ifndef CRG_MAX_DEVICES
#define CRG_MAX_DEVICES 64
#endif
template <bool COUNT, int MINB, int DEFER>
static void launch_trace_variant(const DevScene &sc, const WaveBuffers &wb, int cur, bool sorted, const TraceKnobs &kn, cudaStream_t st) {
	/* launch shape per DEVICE: the host mirror drives several GPUs from one process (one thread each), and both the
	 * occupancy answer and the opt-in shared-memory attribute belong to a device, not to the process */
	struct Shape { int grid; size_t smem; };
	static Shape shapes[CRG_MAX_DEVICES];
	static std::mutex shapes_lock;
	const size_t smem = (size_t)sc.stage_pairs * sizeof(PairNode);
	int dev = 0;
	cudaGetDevice(&dev);
	int grid;
	{
		std::lock_guard<std::mutex> guard(shapes_lock);
		Shape &sh = shapes[dev >= 0 && dev < CRG_MAX_DEVICES ? dev : 0];
		if (!sh.grid || sh.smem != smem) {
			int sms = 0, occ = 0;
			cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
			cudaFuncSetAttribute(k_trace<COUNT, MINB, DEFER>, cudaFuncAttributeMaxDynamicSharedMemorySize, CRG_STAGE_PAIRS * (int)sizeof(PairNode));
			cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, k_trace<COUNT, MINB, DEFER>, 256, smem);
			sh.grid = sms * (occ > 0 ? occ : 1);
			sh.smem = smem;
		}
		grid = sh.grid;
	}
	k_trace<COUNT, MINB, DEFER><<<grid, 256, smem, st>>>(sc, wb, cur, kn.refill, kn.burst, sorted ? 1 : 0, kn.inst_min);
}

/* the frame path's knobs: parsed once per process; out-of-range values fall back to the defaults */
const TraceKnobs &crg_trace_knobs_env(void) {
	static const TraceKnobs kn = [] {
		auto env = [](const char *name, int dflt, int lo, int hi) { const char *e = getenv(name); const int v = e ? atoi(e) : dflt; return v >= lo && v <= hi ? v : dflt; };
		TraceKnobs k;
		k.minb = env("CRGPU_TRACE_MINB", 4, 2, 4);
		k.defer = env("CRGPU_TRACE_DEFER", CRG_DEFER_DEFAULT, 0, 2);
		k.refill = env("CRGPU_TRACE_REFILL", CRG_REFILL, 1, 32);
		k.burst = env("CRGPU_TRACE_BURST", k.defer ? 4 : CRG_NODE_BURST, 1, 1 << 30);
		k.inst_min = env("CRGPU_TRACE_INSTMIN", CRG_INST_MIN, 1, 32);
		return k;
	}();
	return kn;
}

void crg_launch_trace(const DevScene &sc, const WaveBuffers &wb, int cur, bool count, bool sorted, const TraceKnobs &kn, cudaStream_t st) {
	if (count) {
		if (kn.defer == 2) launch_trace_variant<true, 3, 2>(sc, wb, cur, sorted, kn, st);
		else if (kn.defer == 1) launch_trace_variant<true, 3, 1>(sc, wb, cur, sorted, kn, st);
		else launch_trace_variant<true, 3, 0>(sc, wb, cur, sorted, kn, st);
		return;
	}
#define CRG_TRACE_DISPATCH(D) do { \
		if (kn.minb == 4) launch_trace_variant<false, 4, D>(sc, wb, cur, sorted, kn, st); \
		else if (kn.minb == 2) launch_trace_variant<false, 2, D>(sc, wb, cur, sorted, kn, st); \
		else launch_trace_variant<false, 3, D>(sc, wb, cur, sorted, kn, st); } while (0)
	if (kn.defer == 2) CRG_TRACE_DISPATCH(2);
	else if (kn.defer == 1) CRG_TRACE_DISPATCH(1);
	else CRG_TRACE_DISPATCH(0);
#undef CRG_TRACE_DISPATCH
}

/* crgpu_trace_rays: K2's write-back as one record per ray.  A hit record (t, u, v, prim slot) and its instance are written
 * together, so the slot is only followed into slot_poly for an instance index K2 can have written. */
struct TraceRecord { float t, u, v; int inst, poly; unsigned key, prim, pad; };
__global__ void __launch_bounds__(256) k_trace_records(DevScene sc, WaveBuffers wb, unsigned n, TraceRecord *__restrict__ out) {
	for (unsigned i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
		const float4 h = wb.hit[i];
		const int inst = wb.hitInst[i];
		TraceRecord r;
		r.t = h.x; r.u = h.y; r.v = h.z; r.inst = inst; r.prim = __float_as_uint(h.w); r.key = wb.hitKey[i]; r.pad = 0u;
		r.poly = -1;
		if (inst >= 0 && (unsigned)inst < sc.instance_count && sc.instances[inst].kind == CRS_INST_MESH) r.poly = (int)sc.slot_poly[r.prim];
		out[i] = r;
	}
}
void crg_launch_trace_records(const DevScene &sc, const WaveBuffers &wb, unsigned n, void *out, int grid, cudaStream_t st) {
	k_trace_records<<<grid, 256, 0, st>>>(sc, wb, n, static_cast<TraceRecord *>(out));
}
static_assert(sizeof(TraceRecord) == 32, "TraceRecord must match struct crgpu_ray_record (include/crgpu.h)");
