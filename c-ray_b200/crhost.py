"""ctypes binding of libcrhost.so — the host C mirror of c-ray's renderer (c-ray_b200/host/cr_host.h): loadScene,
renderFrame behind the tile dispatcher, multi-GPU groups.  Python is the launcher only (bench, tests, torchrun ranks);
every pixel is computed by libcrgpu.so's kernels, dispatched by the C code."""
import ctypes as C
import os

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(HERE, "libcrhost.so")
ID_BYTES = 128


class Texture8(C.Structure):
    _fields_ = [("width", C.c_uint), ("height", C.c_uint), ("data", C.POINTER(C.c_uint8))]


_lib = None


def lib():
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise RuntimeError(f"{LIB_PATH} is missing — build it with `python -c 'import __graft_entry__ as g; g.build()'`")
        L = C.CDLL(LIB_PATH)
        P = C.c_void_p
        L.newRenderer.restype = P
        L.loadSceneFile.argtypes = [P, C.c_char_p] + [C.c_int] * 4
        L.applySceneConfig.argtypes = [P] + [C.c_int] * 4
        L.prepareGpus.argtypes = [P]
        L.crhostUniqueId.argtypes = [P]
        L.joinRanks.argtypes = [P, P, C.c_int, C.c_int, C.c_int]
        L.renderFrame.argtypes = [P]
        L.renderFrame.restype = C.POINTER(Texture8)
        L.destroyTexture8.argtypes = [C.POINTER(Texture8)]
        L.destroyRenderer.argtypes = [P]
        L.crhostRenderBuffer.argtypes = [P]
        L.crhostRenderBuffer.restype = C.POINTER(C.c_float)
        L.crhostRenderSeconds.argtypes = [P]
        L.crhostRenderSeconds.restype = C.c_double
        L.crhostTotalRays.argtypes = [P]
        L.crhostTotalRays.restype = C.c_ulonglong
        L.crhostConfigure.argtypes = [P, C.c_int, C.c_uint, C.c_uint, C.c_int]
        L.crhostImageSize.argtypes = [P, C.POINTER(C.c_uint), C.POINTER(C.c_uint), C.POINTER(C.c_int), C.POINTER(C.c_int)]
        L.crhostComm.argtypes = [P]
        L.crhostComm.restype = P
        L.crhostPrepared.argtypes = [P]
        L.crhostPrepared.restype = P
        L.crhostTileCount.argtypes = [P]
        L.crhostSetRank.argtypes = [P, C.c_int, C.c_int]
        L.crhostResetQueue.argtypes = [P]
        L.takeRankTiles.argtypes = [P, P, P]
        L.crhostTileOwners.argtypes = [P, C.c_int, P]
        L.crhostTileOwners.restype = None
        L.crhostAbort.argtypes = [P, C.c_int]
        L.crhostAbort.restype = None
        L.crhostSetPaused.argtypes = [P, C.c_int]
        L.crhostSetPaused.restype = None
        L.crhostProgress.argtypes = [P, C.POINTER(C.c_ulonglong)]
        L.crhostWorkerPasses.argtypes = [P, C.c_int]
        L.crhostCurrentImage.argtypes = [P, P]
        L.crhostCurrentImagePasses.argtypes = [P, P, P, C.c_int]
        _lib = L
    return _lib


def unique_id():
    """128-byte NCCL id made by rank 0 of a one-process-per-GPU job; hand it to every rank's Renderer.join()."""
    buf = C.create_string_buffer(ID_BYTES)
    if lib().crhostUniqueId(buf) != 0:
        raise RuntimeError("crhostUniqueId failed (libcrgpu_nccl.so / NCCL not available)")
    return buf.raw


class Renderer:
    """struct renderer of cr_host.h: scene (JSON or .crscene) + prefs + tile queue; render() = renderFrame."""

    def __init__(self, scene_path, width=0, height=0, samples=0, bounces=0, gpus=1, tile=0, quiet=True):
        L = lib()
        self.r = L.newRenderer()
        L.crhostConfigure(self.r, gpus, tile, tile, 1 if quiet else 0)
        if L.loadSceneFile(self.r, os.fsencode(scene_path), width, height, samples, bounces) != 0:
            L.destroyRenderer(self.r)
            self.r = None
            raise RuntimeError(f"loadSceneFile({scene_path}) failed")
        w, h, s, b = C.c_uint(), C.c_uint(), C.c_int(), C.c_int()
        L.crhostImageSize(self.r, C.byref(w), C.byref(h), C.byref(s), C.byref(b))
        self.W, self.H, self.samples, self.bounces = w.value, h.value, s.value, b.value

    def prepare(self):
        """Scene re-layout into pinned host memory + (for gpus > 1) the in-process NCCL group: once, outside the frames."""
        if lib().prepareGpus(self.r) != 0:
            raise RuntimeError("prepareGpus failed (no CUDA device, unsupported scene, or NCCL unavailable)")

    def join(self, uid, rank, world, device):
        if lib().joinRanks(self.r, uid, rank, world, device) != 0:
            raise RuntimeError(f"joinRanks(rank {rank} of {world}, device {device}) failed")

    def render(self):
        """renderFrame: upload -> tiles -> (gather) -> renderBuffer + 8-bit image on the host.  Returns (seconds, rays), or None
        when the frame was aborted without saving (abort(save=False) from another thread)."""
        L = lib()
        self._discard = False
        img = L.renderFrame(self.r)
        if not img:
            if self._discard:
                return None
            raise RuntimeError("renderFrame failed (see stderr)")
        L.destroyTexture8(img)
        return L.crhostRenderSeconds(self.r), int(L.crhostTotalRays(self.r))

    # Controls of a frame in flight (any thread; render() releases the GIL while the frame renders).
    def abort(self, save=True):
        """Stop the frame at a pass boundary; with save, render() returns the committed passes, without it no image."""
        self._discard = not save
        lib().crhostAbort(self.r, 1 if save else 0)

    def set_paused(self, on):
        lib().crhostSetPaused(self.r, 1 if on else 0)

    def progress(self):
        """(whether a frame renders, tile-passes committed by all workers so far)"""
        done = C.c_ulonglong(0)
        busy = lib().crhostProgress(self.r, C.byref(done))
        return bool(busy), int(done.value)

    def worker_passes(self, t):
        """passes worker t has committed in the current (or last) frame: its tiles hold exactly passes [0, that)"""
        return int(lib().crhostWorkerPasses(self.r, t))

    def current_image(self, workers=0):
        """(whether a frame renders, uint8 [H, W, 3] image of the frame as it stands (crhostCurrentImage), and with workers > 0
        the pass count each of the first `workers` workers' tiles show, read together with the image)"""
        img = np.empty((self.H, self.W, 3), dtype=np.uint8)
        passes = np.zeros(max(workers, 1), dtype=np.int32)
        busy = lib().crhostCurrentImagePasses(self.r, img.ctypes.data, passes.ctypes.data if workers else None, workers)
        return bool(busy), img, passes[:workers].tolist()

    def rank_tiles(self, rank, world):
        """(rects (n,4) int32, owner (tileCount,) int32, all_rects (tileCount,4)): this rank's share of the tile queue as the C
        dispatcher assigns it (takeRankTiles), plus every tile's rectangle and owner in queue order."""
        L = lib()
        n = L.crhostTileCount(self.r)
        every = np.zeros((n, 4), dtype=np.int32)
        nums = np.zeros(n, dtype=np.int32)
        L.crhostSetRank(self.r, 0, 1)
        L.crhostResetQueue(self.r)
        assert L.takeRankTiles(self.r, every.ctypes.data, nums.ctypes.data) == n
        rects = np.zeros((n, 4), dtype=np.int32)
        L.crhostSetRank(self.r, rank, world)
        L.crhostResetQueue(self.r)
        got = L.takeRankTiles(self.r, rects.ctypes.data, nums.ctypes.data)
        L.crhostResetQueue(self.r)
        owner = np.zeros(n, dtype=np.int32)
        L.crhostTileOwners(self.r, world, owner.ctypes.data)
        return rects[:got].copy(), owner, every

    def comm(self):
        return lib().crhostComm(self.r)

    def prepared(self):
        return lib().crhostPrepared(self.r)

    def framebuffer(self):
        """numpy view (H, W, 3) fp32 of state.renderBuffer (valid until the renderer is reconfigured or closed)."""
        p = lib().crhostRenderBuffer(self.r)
        return np.ctypeslib.as_array(p, shape=(self.H, self.W, 3))

    def close(self):
        if self.r:
            lib().destroyRenderer(self.r)
            self.r = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass
