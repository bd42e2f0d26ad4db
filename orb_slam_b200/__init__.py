"""orb_slam_b200 -- H100-native ORB feature front-end (extract + match) behind ORB-SLAM's
ORBextractor / ORBmatcher API.  (The package name is historical.)

The product is `liborbfe.so` (hand-written sm_90a CUDA + a C-ABI, see include/orbfe.h) and the C++
facades in orb_slam_b200/host/.  This module is only a thin ctypes binding of the C-ABI used by the
tests and bench.py; it mirrors the reference's class names and argument meaning
(include/ORBextractor.h:32-77, include/ORBmatcher.h:37-107 of raulmur/ORB_SLAM).

There is no CPU fallback: if the shared library is missing the import of `lib()` raises, and on a box
without a CUDA device the constructors raise OrbfeError(ORBFE_ERR_NO_DEVICE).
"""
import ctypes as C
import os

import numpy as np

__all__ = ["ORBextractor", "ORBmatcher", "OrbfeError", "KP_DTYPE", "lib", "library_path", "HARRIS_SCORE", "FAST_SCORE"]

_HERE = os.path.dirname(os.path.abspath(__file__))
_SO = os.path.join(_HERE, "liborbfe.so")

HARRIS_SCORE, FAST_SCORE = 0, 1  # ORBextractor.h:37
ORBFE_OK, ORBFE_ERR_ARG, ORBFE_ERR_UNSUPPORTED, ORBFE_ERR_CAPACITY = 0, -1, -2, -3
ORBFE_ERR_CUDA, ORBFE_ERR_NO_DEVICE, ORBFE_ERR_INTERNAL = -4, -5, -6

# cv::KeyPoint layout (28 bytes)
KP_DTYPE = np.dtype([("x", "<f4"), ("y", "<f4"), ("size", "<f4"), ("angle", "<f4"), ("response", "<f4"),
                     ("octave", "<i4"), ("class_id", "<i4")])

# every symbol include/orbfe.h declares (tests check that the library exports all of them)
ABI_SYMBOLS = [
    "orbfe_last_error", "orbfe_version", "orbfe_device_count",
    "orbfe_extractor_create", "orbfe_extractor_destroy", "orbfe_extractor_levels", "orbfe_extractor_scale_factor",
    "orbfe_extractor_tables", "orbfe_extract", "orbfe_extract_batch", "orbfe_extract_batch_device",
    "orbfe_extractor_sync", "orbfe_extractor_last_launches", "orbfe_extractor_set_profiling", "orbfe_extractor_set_batch_mode",
    "orbfe_extractor_stage_times", "orbfe_debug_level_size", "orbfe_debug_read_level",
    "orbfe_matcher_create", "orbfe_matcher_destroy", "orbfe_hamming_csr", "orbfe_hamming_dense",
    "orbfe_knn2_groups", "orbfe_knn2_groups_device", "orbfe_hamming_csr_device", "orbfe_matcher_sync",
    "orbfe_matcher_counters",
    # include/orbfe_match.h
    "orbfe_frame_scale_factors", "orbfe_search_by_projection_frames", "orbfe_search_by_projection_device", "orbfe_guided_search_device",
    "orbfe_search_for_initialization_device", "orbfe_search_by_bow_device", "orbfe_search_for_triangulation_device",
    "orbfe_search_local_points", "orbfe_search_by_projection_kf",
    "orbfe_search_by_projection_f1f2", "orbfe_search_by_bow", "orbfe_guided_search", "orbfe_guided_best", "orbfe_search_for_triangulation",
    "orbfe_window_search",
    "orbfe_search_for_initialization",
    "orbfe_undistort_keypoints_device", "orbfe_undistort_keypoints", "orbfe_image_bounds",
    # include/orbfe_comm.h
    "orbfe_comm_unique_id", "orbfe_comm_create", "orbfe_comm_destroy", "orbfe_comm_world", "orbfe_comm_rank", "orbfe_comm_nccl_version",
    "orbfe_comm_sync", "orbfe_comm_barrier", "orbfe_allgather_desc", "orbfe_comm_broadcast", "orbfe_comm_allgather", "orbfe_shard_range",
    "orbfe_knn2_sweep_sharded", "orbfe_rig_exchange_create", "orbfe_rig_exchange_destroy", "orbfe_extract_batch_device_exchange",
    "orbfe_rig_exchange_wait", "orbfe_rig_exchange_release", "orbfe_search_for_initialization_exchange", "orbfe_rig_exchange_buffers", "orbfe_rig_exchange_buffers_produced", "orbfe_rig_exchange_check",
    "orbfe_rig_exchange_bytes",
    # include/orbfe_bow.h
    "orbfe_vocabulary_create", "orbfe_vocabulary_destroy", "orbfe_bow_descend_device", "orbfe_bow_descend", "orbfe_bow_transform",
    "orbfe_distinctive_descriptors", "orbfe_bow_db_detect", "orbfe_feature_vector_device", "orbfe_distinctive_descriptors_device",
    "orbfe_bow_vector_device",
    "orbfe_kfdb_create", "orbfe_kfdb_destroy", "orbfe_kfdb_add", "orbfe_kfdb_add_device", "orbfe_kfdb_erase", "orbfe_kfdb_clear", "orbfe_kfdb_set_covisibles",
    "orbfe_kfdb_size", "orbfe_kfdb_detect", "orbfe_kfdb_detect_device",
]


class OrbfeError(RuntimeError):
    def __init__(self, code, msg):
        super().__init__("orbfe error %d: %s" % (code, msg))
        self.code = code


def library_path():
    return _SO


_lib = None


def lib():
    """Load liborbfe.so (built in-tree by orb_slam_b200/build.py). Raises if it is missing: no fallback."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(_SO):
        raise ImportError("liborbfe.so not built: run `python -m orb_slam_b200.build` (nvcc, sm_90a). "
                          "There is no CPU fallback.")
    L = C.CDLL(_SO)
    vp, ip = C.c_void_p, C.POINTER(C.c_int)
    L.orbfe_last_error.restype = C.c_char_p
    L.orbfe_extractor_create.argtypes = [C.c_int, C.c_float, C.c_int, C.c_int, C.c_int, C.c_int, C.POINTER(vp)]
    L.orbfe_extractor_destroy.argtypes = [vp]
    L.orbfe_extractor_set_batch_mode.argtypes = [vp, C.c_int]
    L.orbfe_extractor_levels.argtypes = [vp]
    L.orbfe_extractor_scale_factor.argtypes = [vp]
    L.orbfe_extractor_scale_factor.restype = C.c_float
    L.orbfe_extractor_tables.argtypes = [vp, vp, vp, vp]
    L.orbfe_extract.argtypes = [vp, vp, C.c_int, C.c_int, C.c_size_t, vp, vp, C.c_int, ip]
    L.orbfe_extract_batch.argtypes = [vp, vp, C.c_int, C.c_int, C.c_size_t, C.c_size_t, C.c_int, vp, vp, C.c_int, vp]
    L.orbfe_extract_batch_device.argtypes = [vp, vp, C.c_int, C.c_int, C.c_size_t, C.c_size_t, C.c_int, vp, vp, vp, vp]
    L.orbfe_extractor_sync.argtypes = [vp]
    L.orbfe_extractor_last_launches.argtypes = [vp]
    L.orbfe_extractor_set_profiling.argtypes = [vp, C.c_int]
    L.orbfe_extractor_stage_times.argtypes = [vp, vp, vp, C.c_int]
    L.orbfe_debug_level_size.argtypes = [vp, C.c_int, ip, ip]
    L.orbfe_debug_read_level.argtypes = [vp, C.c_int, C.c_int, C.c_int, vp, C.c_size_t]
    L.orbfe_matcher_create.argtypes = [C.c_int, C.POINTER(vp)]
    L.orbfe_matcher_destroy.argtypes = [vp]
    L.orbfe_hamming_csr.argtypes = [vp, vp, C.c_int, vp, C.c_int, vp, vp, vp]
    L.orbfe_hamming_dense.argtypes = [vp, vp, C.c_int, vp, C.c_int, vp]
    L.orbfe_knn2_groups.argtypes = [vp, vp, C.c_int, vp, C.c_int, C.c_int, vp, vp, vp]
    L.orbfe_knn2_groups_device.argtypes = [vp, vp, C.c_int, vp, C.c_int, C.c_int, vp, vp, vp, vp]
    L.orbfe_hamming_csr_device.argtypes = [vp, vp, vp, vp, vp, C.c_int, C.c_int, vp, vp]
    L.orbfe_matcher_sync.argtypes = [vp]
    L.orbfe_matcher_counters.argtypes = [vp, vp, vp, vp]
    _lib = L
    return L


def _check(rc):
    if rc != 0:
        raise OrbfeError(rc, lib().orbfe_last_error().decode("utf-8", "replace"))


def _p(a):
    return a.ctypes.data_as(C.c_void_p) if a is not None else None


class ORBextractor:
    """Mirror of ORB_SLAM::ORBextractor (ctor: src/ORBextractor.cc:457-511; operator(): :718-779).

    ORBextractor(nfeatures=1000, scaleFactor=1.2, nlevels=8, scoreType=FAST_SCORE, fastTh=20)
    """

    def __init__(self, nfeatures=1000, scaleFactor=1.2, nlevels=8, scoreType=FAST_SCORE, fastTh=20, device=0):
        self._h = C.c_void_p()
        self.nfeatures = nfeatures
        _check(lib().orbfe_extractor_create(nfeatures, scaleFactor, nlevels, scoreType, fastTh, device, C.byref(self._h)))
        self.nlevels = nlevels

    def close(self):
        if getattr(self, "_h", None) and self._h.value:
            lib().orbfe_extractor_destroy(self._h)
            self._h = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    @property
    def handle(self):
        return self._h

    def GetLevels(self):
        return lib().orbfe_extractor_levels(self._h)

    def GetScaleFactor(self):
        return lib().orbfe_extractor_scale_factor(self._h)

    def tables(self):
        n = self.nlevels
        s, i, q = np.zeros(n, np.float32), np.zeros(n, np.float32), np.zeros(n, np.int32)
        _check(lib().orbfe_extractor_tables(self._h, _p(s), _p(i), _p(q)))
        return s, i, q

    def __call__(self, image, mask=None, cap=None):
        """operator()(image, mask, keypoints, descriptors): returns (keypoints[KP_DTYPE], descriptors[N,32]).

        `mask` is accepted for signature parity and must be empty (Frame.cc:60 always passes cv::Mat())."""
        if mask is not None and getattr(mask, "size", 0):
            raise OrbfeError(ORBFE_ERR_UNSUPPORTED, "non-empty mask is outside the hot path (Frame.cc:60 passes an empty Mat)")
        if image is None or image.size == 0:
            return np.zeros(0, KP_DTYPE), np.zeros((0, 32), np.uint8)
        assert image.dtype == np.uint8 and image.ndim == 2, "CV_8UC1 expected (ORBextractor.cc:725)"
        if image.strides[1] != 1:
            image = np.ascontiguousarray(image)
        H, W = image.shape
        cap = cap or max(self.nfeatures, 1)
        kps = np.zeros(cap, KP_DTYPE)
        desc = np.zeros((cap, 32), np.uint8)
        n = C.c_int(0)
        _check(lib().orbfe_extract(self._h, _p(image), W, H, image.strides[0], _p(kps), _p(desc), cap, C.byref(n)))
        return kps[:n.value], desc[:n.value]

    def extract_batch(self, images, cap=None):
        """images: uint8 array [B, H, W] (C-contiguous rows). Returns (kps[B,cap], desc[B,cap,32], counts[B])."""
        assert images.dtype == np.uint8 and images.ndim == 3 and images.strides[2] == 1
        B, H, W = images.shape
        cap = cap or max(self.nfeatures, 1)
        kps = np.zeros((B, cap), KP_DTYPE)
        desc = np.zeros((B, cap, 32), np.uint8)
        counts = np.zeros(B, np.int32)
        _check(lib().orbfe_extract_batch(self._h, _p(images), W, H, images.strides[1], images.strides[0], B,
                                         _p(kps), _p(desc), cap, _p(counts)))
        return kps, desc, counts

    def extract_batch_ptr(self, host_ptr, W, H, stride, frame_stride, B, kps_ptr, desc_ptr, cap, counts_ptr):
        """Raw-pointer form of orbfe_extract_batch (pinned host buffers owned by the caller)."""
        _check(lib().orbfe_extract_batch(self._h, C.c_void_p(host_ptr), W, H, stride, frame_stride, B,
                                         C.c_void_p(kps_ptr), C.c_void_p(desc_ptr), cap, C.c_void_p(counts_ptr)))

    def extract_batch_device(self, d_imgs, W, H, stride, frame_stride, B, d_kps, d_desc, d_counts, stream=0):
        """Device-pointer form (ints = raw device addresses); enqueues on `stream`, does not synchronise."""
        _check(lib().orbfe_extract_batch_device(self._h, C.c_void_p(d_imgs), W, H, stride, frame_stride, B,
                                                C.c_void_p(d_kps), C.c_void_p(d_desc), C.c_void_p(d_counts),
                                                C.c_void_p(stream)))

    def set_batch_mode(self, mode):
        """0 = chunked (one handle), 1 = phased (two alternating handles); see include/orbfe.h."""
        _check(lib().orbfe_extractor_set_batch_mode(self._h, int(mode)))

    def sync(self):
        _check(lib().orbfe_extractor_sync(self._h))

    def last_launches(self):
        return lib().orbfe_extractor_last_launches(self._h)

    def set_profiling(self, on):
        _check(lib().orbfe_extractor_set_profiling(self._h, int(on)))

    def stage_times(self):
        cap = 32768   # the library keeps at most 16384 intervals between two reads
        names = (C.c_char * 32 * cap)()
        ms = (C.c_float * cap)()
        n = lib().orbfe_extractor_stage_times(self._h, names, ms, cap)
        return [(names[i].value.decode(), ms[i]) for i in range(n)]

    def debug_level(self, frame, level, blurred=False):
        w, h = C.c_int(), C.c_int()
        _check(lib().orbfe_debug_level_size(self._h, level, C.byref(w), C.byref(h)))
        out = np.empty((h.value, w.value), np.uint8)
        _check(lib().orbfe_debug_read_level(self._h, frame, level, int(blurred), _p(out), out.strides[0]))
        return out


class ORBmatcher:
    """Device half of ORB_SLAM::ORBmatcher (src/ORBmatcher.cc): batched 256-bit Hamming distances.

    The sequential accept/skip logic of each Search* routine stays on the host (C++ facade in
    orb_slam_b200/host/ORBmatcher.cc; Python replays for the tests live in orb_slam_b200/matching.py).
    """
    TH_LOW, TH_HIGH, HISTO_LENGTH = 50, 100, 30  # ORBmatcher.cc:40-42

    def __init__(self, nnratio=0.6, checkOri=True, device=0):
        self.mfNNratio = np.float32(nnratio)
        self.mbCheckOrientation = bool(checkOri)
        self._h = C.c_void_p()
        _check(lib().orbfe_matcher_create(device, C.byref(self._h)))

    def close(self):
        if getattr(self, "_h", None) and self._h.value:
            lib().orbfe_matcher_destroy(self._h)
            self._h = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    @property
    def handle(self):
        return self._h

    def hamming_csr(self, qdesc, tdesc, row_ptr, cols):
        qdesc = np.ascontiguousarray(qdesc, np.uint8)
        tdesc = np.ascontiguousarray(tdesc, np.uint8)
        row_ptr = np.ascontiguousarray(row_ptr, np.int32)
        cols = np.ascontiguousarray(cols, np.int32)
        out = np.zeros(len(cols), np.uint16)
        _check(lib().orbfe_hamming_csr(self._h, _p(qdesc), qdesc.shape[0], _p(tdesc), tdesc.shape[0], _p(row_ptr),
                                       _p(cols), _p(out)))
        return out

    def hamming_dense(self, qdesc, tdesc):
        qdesc = np.ascontiguousarray(qdesc, np.uint8)
        tdesc = np.ascontiguousarray(tdesc, np.uint8)
        out = np.zeros((qdesc.shape[0], tdesc.shape[0]), np.uint16)
        _check(lib().orbfe_hamming_dense(self._h, _p(qdesc), qdesc.shape[0], _p(tdesc), tdesc.shape[0], _p(out)))
        return out

    def knn2_groups(self, qdesc, db, group_size):
        qdesc = np.ascontiguousarray(qdesc, np.uint8)
        db = np.ascontiguousarray(db, np.uint8)
        assert db.shape[0] % group_size == 0
        ng, nq = db.shape[0] // group_size, qdesc.shape[0]
        best = np.zeros((ng, nq), np.uint16)
        idx = np.zeros((ng, nq), np.int32)
        second = np.zeros((ng, nq), np.uint16)
        _check(lib().orbfe_knn2_groups(self._h, _p(qdesc), nq, _p(db), ng, group_size, _p(best), _p(idx), _p(second)))
        return best, idx, second

    def sync(self):
        _check(lib().orbfe_matcher_sync(self._h))

    def counters(self):
        """(h2d_bytes, d2h_bytes, launches) accumulated by the host-pointer entry points."""
        a, b, c = C.c_ulonglong(), C.c_ulonglong(), C.c_ulonglong()
        _check(lib().orbfe_matcher_counters(self._h, C.byref(a), C.byref(b), C.byref(c)))
        return a.value, b.value, c.value
