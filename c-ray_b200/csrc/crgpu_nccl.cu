/*
 * crgpu_nccl.cu — framebuffer tile gather over NCCL (include/crgpu_nccl.h).  Plumbing only: tiles are packed by a copy
 * kernel per sender, exchanged with grouped ncclSend/ncclRecv and unpacked by a copy kernel per peer on the root (one launch
 * per 32,768 tiles); no arithmetic touches the pixels.
 */
#include "../../include/crgpu_nccl.h"
#include <cuda_runtime.h>
#include <nccl.h>
#include <vector>
#include <cstdio>
#include <cstring>

struct Member {                  /* one GPU of the group that lives in THIS process */
	int device = 0;
	int rank = 0;
	ncclComm_t comm = nullptr;
	cudaStream_t stream = nullptr;
	float *stage = nullptr; size_t stage_cap = 0;       /* packed tiles of this member (send side) */
	int4 *tiles = nullptr; size_t tiles_cap = 0;        /* device tile list: (x0, y0, x1, y1) */
	unsigned long long *offs = nullptr;                 /* device: float offset of each tile inside the packed buffer */
	std::vector<float *> recv;                           /* root only: one buffer per peer */
	std::vector<size_t> recv_cap;
	std::vector<unsigned long long> list_key;            /* per group member: fingerprint of its tile list as last uploaded to tiles/offs */
	cudaStream_t own_stream = nullptr;
};

struct crgpu_comm {
	int world = 0;
	std::vector<Member> members;     /* in-process: world members; rank mode: exactly one */
	bool rank_mode = false;
};

#define NCHECK(x) do { ncclResult_t r_ = (x); if (r_ != ncclSuccess) { fprintf(stderr, "crgpu_nccl: %s: %s\n", #x, ncclGetErrorString(r_)); return CRGPU_ERR_CUDA; } } while (0)
#define CCHECK(x) do { cudaError_t e_ = (x); if (e_ != cudaSuccess) { fprintf(stderr, "crgpu_nccl: %s: %s\n", #x, cudaGetErrorString(e_)); return CRGPU_ERR_CUDA; } } while (0)

/* blockIdx.y = tile; the block's threads walk the tile's floats.  Framebuffer rows: y0..y1-1 (y up) are storage rows H-y1..H-1-y0. */
template <bool PACK>
__global__ void k_tiles_copy(float *__restrict__ fb, float *__restrict__ packed, const int4 *__restrict__ tiles,
							  const unsigned long long *__restrict__ offs, int W, int H) {
	const int4 r = tiles[blockIdx.y];
	const unsigned roww = (unsigned)(r.z - r.x) * 3u;
	const unsigned n = roww * (unsigned)(r.w - r.y);
	float *p = packed + offs[blockIdx.y];
	for (unsigned i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
		const unsigned row = i / roww, col = i - row * roww;
		float *f = fb + ((size_t)(H - r.w + (int)row) * (size_t)W + (size_t)r.x) * 3u + col;
		if (PACK) p[i] = *f; else *f = p[i];
	}
}

static inline size_t tile_floats(const int *r) { return (size_t)(r[2] - r[0]) * (size_t)(r[3] - r[1]) * 3u; }

static int reserve(Member &m, size_t stage_floats, size_t ntiles) {
	if (stage_floats > m.stage_cap) {
		if (m.stage) cudaFree(m.stage);
		m.stage = nullptr; m.stage_cap = 0;
		CCHECK(cudaMalloc((void **)&m.stage, stage_floats * sizeof(float)));
		m.stage_cap = stage_floats;
	}
	if (ntiles > m.tiles_cap) {
		if (m.tiles) cudaFree(m.tiles);
		if (m.offs) cudaFree(m.offs);
		m.tiles = nullptr; m.offs = nullptr; m.tiles_cap = 0;
		CCHECK(cudaMalloc((void **)&m.tiles, ntiles * sizeof(int4)));
		CCHECK(cudaMalloc((void **)&m.offs, ntiles * sizeof(unsigned long long)));
		m.tiles_cap = ntiles;
		m.list_key.clear();
	}
	return CRGPU_OK;
}

/* launch one copy kernel over the tiles of `who` (selected from rects/owner), between fb and `packed`, on m.stream */
template <bool PACK>
static int copy_tiles(Member &m, float *fb, float *packed, const int *rects, const int *owner, int ntiles, int who, int W, int H, size_t slot) {
	std::vector<int4> t;
	std::vector<unsigned long long> o;
	unsigned long long off = 0;
	for (int i = 0; i < ntiles; ++i) {
		if (owner[i] != who) continue;
		const int *r = rects + 4 * i;
		t.push_back(make_int4(r[0], r[1], r[2], r[3]));
		o.push_back(off);
		off += tile_floats(r);
	}
	if (t.empty()) return CRGPU_OK;
	/* The device tile lists change only when the tile grid or the assignment does: fingerprint what was uploaded per member and
	 * skip the (synchronising) upload when it is the same list at the same slot — the steady state of a multi-frame job. */
	unsigned long long key = 1469598103934665603ull ^ (unsigned long long)slot;
	for (const int4 &q : t) { const unsigned v[4] = { (unsigned)q.x, (unsigned)q.y, (unsigned)q.z, (unsigned)q.w }; for (unsigned x : v) key = (key ^ x) * 1099511628211ull; }
	key = (key ^ (unsigned long long)t.size()) * 1099511628211ull;
	if (m.list_key.size() <= (size_t)who) m.list_key.resize((size_t)who + 1, 0ull);
	if (m.list_key[(size_t)who] != key) {
		CCHECK(cudaMemcpyAsync(m.tiles + slot, t.data(), t.size() * sizeof(int4), cudaMemcpyHostToDevice, m.stream));
		CCHECK(cudaMemcpyAsync(m.offs + slot, o.data(), o.size() * sizeof(unsigned long long), cudaMemcpyHostToDevice, m.stream));
		CCHECK(cudaStreamSynchronize(m.stream));                    /* t and o are pageable locals */
		m.list_key[(size_t)who] = key;
	}
	/* gridDim.y <= 65535: an 8K frame in 8x8 tiles on two GPUs is 259,200 tiles per peer.  offs are offsets into the whole
	 * packed buffer, so a chunk only moves its view of the two lists. */
	for (size_t first = 0; first < t.size(); first += 32768u) {
		const size_t cnt = t.size() - first < 32768u ? t.size() - first : 32768u;
		k_tiles_copy<PACK><<<dim3(4, (unsigned)cnt), 256, 0, m.stream>>>(fb, packed, m.tiles + slot + first, m.offs + slot + first, W, H);
		CCHECK(cudaGetLastError());
	}
	return CRGPU_OK;
}

extern "C" int crgpu_comm_create(const int *devices, int n, crgpu_comm **out) {
	if (!devices || !out || n < 1) return CRGPU_ERR_BAD_ARGUMENT;
	crgpu_comm *c = new crgpu_comm();
	c->world = n;
	c->members.resize((size_t)n);
	std::vector<ncclComm_t> comms((size_t)n);
	std::vector<int> devs(devices, devices + n);
	NCHECK(ncclCommInitAll(comms.data(), n, devs.data()));
	for (int i = 0; i < n; ++i) {
		Member &m = c->members[(size_t)i];
		m.device = devices[i]; m.rank = i; m.comm = comms[(size_t)i];
		CCHECK(cudaSetDevice(m.device));
		CCHECK(cudaStreamCreateWithFlags(&m.stream, cudaStreamNonBlocking));
		m.own_stream = m.stream;
		m.recv.assign((size_t)n, nullptr); m.recv_cap.assign((size_t)n, 0);
	}
	*out = c;
	return CRGPU_OK;
}

extern "C" int crgpu_comm_unique_id(void *id_out) {
	if (!id_out) return CRGPU_ERR_BAD_ARGUMENT;
	static_assert(sizeof(ncclUniqueId) == CRGPU_COMM_ID_BYTES, "ncclUniqueId is 128 bytes");
	ncclUniqueId id;
	NCHECK(ncclGetUniqueId(&id));
	memcpy(id_out, &id, sizeof id);
	return CRGPU_OK;
}

extern "C" int crgpu_comm_create_rank(const void *id, int rank, int world, int device, crgpu_comm **out) {
	if (!id || !out || world < 1 || rank < 0 || rank >= world) return CRGPU_ERR_BAD_ARGUMENT;
	crgpu_comm *c = new crgpu_comm();
	c->world = world; c->rank_mode = true;
	c->members.resize(1);
	Member &m = c->members[0];
	m.device = device; m.rank = rank;
	CCHECK(cudaSetDevice(device));
	ncclUniqueId uid;
	memcpy(&uid, id, sizeof uid);
	NCHECK(ncclCommInitRank(&m.comm, world, uid, rank));
	CCHECK(cudaStreamCreateWithFlags(&m.stream, cudaStreamNonBlocking));
	m.own_stream = m.stream;
	m.recv.assign((size_t)world, nullptr); m.recv_cap.assign((size_t)world, 0);
	*out = c;
	return CRGPU_OK;
}

/* shared by both modes: `local` lists the members of this process, fb[k] the framebuffer of local[k] */
static int gather(crgpu_comm *c, std::vector<Member *> &local, std::vector<float *> &fb, int W, int H,
				  const int *rects, const int *owner, int ntiles, int root) {
	const int world = c->world;
	std::vector<size_t> total((size_t)world, 0), count((size_t)world, 0);
	for (int t = 0; t < ntiles; ++t) {
		if (owner[t] < 0 || owner[t] >= world) return CRGPU_ERR_BAD_ARGUMENT;
		const int *r = rects + 4 * t;
		if (r[0] < 0 || r[1] < 0 || r[2] > W || r[3] > H || r[2] <= r[0] || r[3] <= r[1]) return CRGPU_ERR_BAD_ARGUMENT;
		total[(size_t)owner[t]] += tile_floats(r);
		count[(size_t)owner[t]]++;
	}
	Member *rootm = nullptr; float *rootfb = nullptr;
	for (size_t k = 0; k < local.size(); ++k) if (local[k]->rank == root) { rootm = local[k]; rootfb = fb[k]; }
	/* senders: pack */
	for (size_t k = 0; k < local.size(); ++k) {
		Member &m = *local[k];
		if (m.rank == root || total[(size_t)m.rank] == 0) continue;
		CCHECK(cudaSetDevice(m.device));
		int rc = reserve(m, total[(size_t)m.rank], count[(size_t)m.rank]);
		if (rc) return rc;
		rc = copy_tiles<true>(m, fb[k], m.stage, rects, owner, ntiles, m.rank, W, H, 0);
		if (rc) return rc;
	}
	/* root: receive buffers + room for every peer's tile list */
	if (rootm) {
		CCHECK(cudaSetDevice(rootm->device));
		int rc = reserve(*rootm, 0, (size_t)ntiles);
		if (rc) return rc;
		for (int i = 0; i < world; ++i) {
			if (i == root || total[(size_t)i] <= rootm->recv_cap[(size_t)i]) continue;
			if (rootm->recv[(size_t)i]) cudaFree(rootm->recv[(size_t)i]);
			rootm->recv[(size_t)i] = nullptr; rootm->recv_cap[(size_t)i] = 0;
			CCHECK(cudaMalloc((void **)&rootm->recv[(size_t)i], total[(size_t)i] * sizeof(float)));
			rootm->recv_cap[(size_t)i] = total[(size_t)i];
		}
	}
	/* one grouped exchange: every peer sends its packed tiles to the root */
	NCHECK(ncclGroupStart());
	for (Member *m : local) {
		if (m->rank == root || total[(size_t)m->rank] == 0) continue;
		NCHECK(ncclSend(m->stage, total[(size_t)m->rank], ncclFloat, root, m->comm, m->stream));
	}
	if (rootm)
		for (int i = 0; i < world; ++i) {
			if (i == root || total[(size_t)i] == 0) continue;
			NCHECK(ncclRecv(rootm->recv[(size_t)i], total[(size_t)i], ncclFloat, i, rootm->comm, rootm->stream));
		}
	NCHECK(ncclGroupEnd());
	/* root: unpack */
	if (rootm) {
		CCHECK(cudaSetDevice(rootm->device));
		size_t slot = 0;
		for (int i = 0; i < world; ++i) {
			if (i == root || total[(size_t)i] == 0) continue;
			int rc = copy_tiles<false>(*rootm, rootfb, rootm->recv[(size_t)i], rects, owner, ntiles, i, W, H, slot);
			if (rc) return rc;
			slot += count[(size_t)i];
		}
	}
	for (Member *m : local) { CCHECK(cudaSetDevice(m->device)); CCHECK(cudaStreamSynchronize(m->stream)); }
	return CRGPU_OK;
}

extern "C" int crgpu_comm_gather_tiles(crgpu_comm *c, crgpu_scene **scenes, const int *rects, const int *owner, int ntiles, int root) {
	if (!c || c->rank_mode || !scenes || !rects || !owner || root < 0 || root >= c->world) return CRGPU_ERR_BAD_ARGUMENT;
	std::vector<Member *> local;
	std::vector<float *> fb;
	int W = 0, H = 0;
	for (int i = 0; i < c->world; ++i) {
		int dev = -1, w = 0, h = 0;
		void *p = nullptr;
		if (crgpu_scene_info(scenes[i], &dev, &w, &h) || crgpu_framebuffer_device_ptr(scenes[i], &p, nullptr)) return CRGPU_ERR_BAD_ARGUMENT;
		if (dev != c->members[(size_t)i].device) return CRGPU_ERR_BAD_ARGUMENT;
		if (i == 0) { W = w; H = h; } else if (w != W || h != H) return CRGPU_ERR_BAD_ARGUMENT;
		local.push_back(&c->members[(size_t)i]);
		fb.push_back(static_cast<float *>(p));
	}
	return gather(c, local, fb, W, H, rects, owner, ntiles, root);
}

extern "C" int crgpu_comm_gather_tiles_rank(crgpu_comm *c, crgpu_scene *mine, const int *rects, const int *owner, int ntiles, int root) {
	if (!c || !c->rank_mode || !mine || !rects || !owner || root < 0 || root >= c->world) return CRGPU_ERR_BAD_ARGUMENT;
	int dev = -1, W = 0, H = 0;
	void *p = nullptr;
	if (crgpu_scene_info(mine, &dev, &W, &H) || crgpu_framebuffer_device_ptr(mine, &p, nullptr)) return CRGPU_ERR_BAD_ARGUMENT;
	if (dev != c->members[0].device) return CRGPU_ERR_BAD_ARGUMENT;
	std::vector<Member *> local(1, &c->members[0]);
	std::vector<float *> fb(1, static_cast<float *>(p));
	return gather(c, local, fb, W, H, rects, owner, ntiles, root);
}

extern "C" int crgpu_comm_set_stream(crgpu_comm *c, void *cuda_stream, int use_own) {
	if (!c || !c->rank_mode) return CRGPU_ERR_BAD_ARGUMENT;
	Member &m = c->members[0];
	CCHECK(cudaSetDevice(m.device));
	CCHECK(cudaStreamSynchronize(m.stream));
	m.stream = use_own ? m.own_stream : static_cast<cudaStream_t>(cuda_stream);
	return CRGPU_OK;
}

extern "C" int crgpu_comm_destroy(crgpu_comm *c) {
	if (!c) return CRGPU_OK;
	for (Member &m : c->members) {
		cudaSetDevice(m.device);
		if (m.stage) cudaFree(m.stage);
		if (m.tiles) cudaFree(m.tiles);
		if (m.offs) cudaFree(m.offs);
		for (float *r : m.recv) if (r) cudaFree(r);
		if (m.own_stream) cudaStreamDestroy(m.own_stream);
		if (m.comm) ncclCommDestroy(m.comm);
	}
	delete c;
	return CRGPU_OK;
}
