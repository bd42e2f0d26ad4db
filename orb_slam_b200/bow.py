"""ctypes wrappers of include/orbfe_bow.h: the DBoW2 vocabulary-tree transform (reference
Thirdparty/DBoW2/DBoW2/TemplatedVocabulary.h:1126-1262; callers Frame.cc:280-287, KeyFrame.cc:56-65) and the batched
MapPoint::ComputeDistinctiveDescriptors (reference src/MapPoint.cc:185-250).  No CPU fallback: every call runs the
CUDA kernels of liborbfe.so."""
import ctypes as C

import numpy as np

from . import ORBmatcher, OrbfeError, lib

TF_IDF, TF, IDF, BINARY = 0, 1, 2, 3
NORM_NONE, NORM_L1, NORM_L2 = 0, 1, 2

_bound = False


def _bind():
    global _bound
    L = lib()
    if _bound:
        return L
    vp = C.c_void_p
    L.orbfe_vocabulary_create.argtypes = [C.c_int, C.c_int, C.c_int, vp, vp, vp, vp, vp, C.c_int, C.c_int]
    L.orbfe_vocabulary_create.restype = vp
    L.orbfe_vocabulary_destroy.argtypes = [vp]
    L.orbfe_vocabulary_destroy.restype = None
    L.orbfe_bow_descend_device.argtypes = [vp, vp, C.c_int, C.c_int, vp, vp, vp]
    L.orbfe_bow_descend.argtypes = [vp, vp, C.c_int, C.c_int, vp, vp]
    L.orbfe_bow_transform.argtypes = [vp, vp, C.c_int, C.c_int, vp, vp, vp, vp, vp, vp, vp]
    L.orbfe_distinctive_descriptors.argtypes = [vp, vp, vp, C.c_int, vp]
    L.orbfe_bow_db_detect.argtypes = [vp, C.c_int, C.c_int, vp, vp, C.c_int, vp, vp, vp, vp, vp, vp, C.c_float, vp, vp, vp, vp]
    L.orbfe_feature_vector_device.argtypes = [vp, C.c_int, vp, vp, vp, C.c_int, vp, vp, vp, vp, vp]
    L.orbfe_bow_vector_device.argtypes = [vp, C.c_int, vp, vp, C.c_int, vp, vp, vp, vp]
    L.orbfe_distinctive_descriptors_device.argtypes = [vp, C.c_int, vp, vp, C.c_int, C.c_int, vp, vp, C.c_int, vp, vp, vp]
    _bound = True
    return L


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


def _check(rc):
    if rc != 0:
        raise OrbfeError(rc, lib().orbfe_last_error().decode("utf-8", "replace") or "bow call failed")


class Vocabulary:
    """The node table of a DBoW2 vocabulary in device memory.  `voc` = dict(node_desc [nnodes,32] u8, child_ptr
    [nnodes+1] i32, children i32, word_id [nnodes] i32, weight [nnodes] f64, L)."""

    def __init__(self, voc, weighting=TF_IDF, norm=NORM_L1, device=0):
        L = _bind()
        a = lambda x, t: np.ascontiguousarray(x, t)
        self.arrays = {k: a(voc[k], t) for k, t in (("node_desc", np.uint8), ("child_ptr", np.int32), ("children", np.int32),
                                                    ("word_id", np.int32), ("weight", np.float64))}
        A = self.arrays
        self._h = L.orbfe_vocabulary_create(device, len(A["word_id"]), int(voc["L"]), _p(A["node_desc"]), _p(A["child_ptr"]),
                                            _p(A["children"]), _p(A["word_id"]), _p(A["weight"]), weighting, norm)
        if not self._h:
            raise OrbfeError(-1, L.orbfe_last_error().decode("utf-8", "replace"))

    @property
    def handle(self):
        return self._h

    def close(self):
        if self._h:
            lib().orbfe_vocabulary_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def descend(self, desc, levelsup=4):
        """Per-descriptor (leaf node id, node id at level L - levelsup)."""
        desc = np.ascontiguousarray(desc, np.uint8).reshape(-1, 32)
        n = len(desc)
        leaf, node = np.zeros(max(n, 1), np.int32), np.zeros(max(n, 1), np.int32)
        _check(_bind().orbfe_bow_descend(self._h, _p(desc), n, levelsup, _p(leaf), _p(node)))
        return leaf[:n], node[:n]

    def descend_device(self, d_desc, n, levelsup, d_leaf, d_node, stream=0):
        """Device-pointer form (ints = raw device addresses); enqueued, not synchronised."""
        vp = C.c_void_p
        _check(_bind().orbfe_bow_descend_device(self._h, vp(d_desc), n, levelsup, vp(d_leaf), vp(d_node), vp(stream)))

    def transform(self, desc, levelsup=4):
        """(BowVector as (word ids, values)), (FeatureVector as CSR (node ids, ptr, feature indices))."""
        desc = np.ascontiguousarray(desc, np.uint8).reshape(-1, 32)
        n = len(desc)
        cap = max(n, 1)
        bow_ids, bow_vals = np.zeros(cap, np.int32), np.zeros(cap, np.float64)
        fv_ids, fv_ptr, fv_feats = np.zeros(cap, np.int32), np.zeros(cap + 1, np.int32), np.zeros(cap, np.int32)
        nw, nn = C.c_int(0), C.c_int(0)
        _check(_bind().orbfe_bow_transform(self._h, _p(desc), n, levelsup, C.byref(nw), _p(bow_ids), _p(bow_vals), C.byref(nn),
                                           _p(fv_ids), _p(fv_ptr), _p(fv_feats)))
        return (bow_ids[:nw.value], bow_vals[:nw.value]), (fv_ids[:nn.value], fv_ptr[:nn.value + 1], fv_feats[:fv_ptr[nn.value]])


def feature_vector_device(voc: "Vocabulary", nframes, d_leaf, d_node, d_counts, cap, d_fv_ids, d_fv_ptr, d_fv_items, d_fv_n, stream=0):
    """FeatureVectors of `nframes` frames from the leaf / node ids Vocabulary.descend_device wrote (ints = raw device addresses;
    frame f at f*cap, d_counts[f] features).  Outputs: node ids (nframes x cap), row starts (nframes x (cap+1)), feature
    indices (nframes x cap), node counts (nframes).  Enqueued, not synchronised; see include/orbfe_bow.h."""
    vp = C.c_void_p
    _check(_bind().orbfe_feature_vector_device(voc.handle, nframes, vp(d_leaf), vp(d_node), vp(d_counts), cap, vp(d_fv_ids),
                                               vp(d_fv_ptr), vp(d_fv_items), vp(d_fv_n), vp(stream)))


def bow_vector_device(voc: "Vocabulary", nframes, d_leaf, d_counts, cap, d_bow_ids, d_bow_vals, d_bow_n, stream=0):
    """BowVectors of `nframes` frames from the leaf ids Vocabulary.descend_device wrote (ints = raw device addresses; frame f
    at f*cap, d_counts[f] features).  Outputs: word ids (nframes x cap, int32), values (nframes x cap, float64), word counts
    (nframes); entries past a frame's word count hold id INT32_MAX and value 0.  Enqueued, not synchronised; see
    include/orbfe_bow.h."""
    vp = C.c_void_p
    _check(_bind().orbfe_bow_vector_device(voc.handle, nframes, vp(d_leaf), vp(d_counts), cap, vp(d_bow_ids), vp(d_bow_vals), vp(d_bow_n),
                                           vp(stream)))


def distinctive_descriptors(matcher: ORBmatcher, desc, group_ptr):
    """Index (inside its group) of the least-median-distance descriptor of every group (map point)."""
    desc = np.ascontiguousarray(desc, np.uint8).reshape(-1, 32)
    group_ptr = np.ascontiguousarray(group_ptr, np.int32)
    ng = len(group_ptr) - 1
    best = np.zeros(max(ng, 1), np.int32)
    _check(_bind().orbfe_distinctive_descriptors(matcher.handle, _p(desc), _p(group_ptr), ng, _p(best)))
    return best[:ng]


def distinctive_descriptors_device(matcher: ORBmatcher, ngroups, d_desc, d_counts, nframes, cap, d_group_ptr, d_obs, nobs, d_best,
                                   d_mp_desc, stream=0):
    """Device-pointer form (ints = raw device addresses) on the frame store: group g owns the observation slots
    d_obs[d_group_ptr[g] .. d_group_ptr[g+1]) (f*cap + i each); d_best[g] receives the chosen position inside the group and
    row g of d_mp_desc (ngroups x 32 bytes) the chosen descriptor.  Enqueued, not synchronised; see include/orbfe_bow.h."""
    vp = C.c_void_p
    _check(_bind().orbfe_distinctive_descriptors_device(matcher.handle, ngroups, vp(d_desc), vp(d_counts), nframes, cap, vp(d_group_ptr),
                                                        vp(d_obs), nobs, vp(d_best), vp(d_mp_desc), vp(stream)))


def db_detect(matcher: ORBmatcher, mode, q_ids, q_vals, kf_ptr, db_ids, db_vals, connected, covis_ptr, covis, min_score=0.0):
    """KeyFrameDatabase::DetectLoopCandidates (mode 0) / DetectRelocalisationCandidates (mode 1) on arrays
    (reference src/KeyFrameDatabase.cc:73-308).  Returns (candidate keyframe indices, shared-word counts, scores)."""
    a = lambda x, t: np.ascontiguousarray(x, t)
    q_ids, q_vals, kf_ptr = a(q_ids, np.int32), a(q_vals, np.float64), a(kf_ptr, np.int32)
    db_ids, db_vals, covis_ptr, covis = a(db_ids, np.int32), a(db_vals, np.float64), a(covis_ptr, np.int32), a(covis, np.int32)
    connected = a(connected, np.uint8)
    nkf = len(kf_ptr) - 1
    cand, common, score = np.zeros(max(nkf, 1), np.int32), np.zeros(max(nkf, 1), np.int32), np.zeros(max(nkf, 1), np.float32)
    nc = C.c_int(0)
    _check(_bind().orbfe_bow_db_detect(matcher.handle, mode, len(q_ids), _p(q_ids), _p(q_vals), nkf, _p(kf_ptr), _p(db_ids), _p(db_vals),
                                       _p(connected), _p(covis_ptr), _p(covis), min_score, C.byref(nc), _p(cand), _p(common), _p(score)))
    return cand[:nc.value], common[:nkf], score[:nkf]


_kfdb_bound = False


def _bind_kfdb():
    global _kfdb_bound
    L = _bind()
    if _kfdb_bound:
        return L
    vp, i = C.c_void_p, C.c_int
    L.orbfe_kfdb_create.argtypes = [vp, i, C.c_longlong, C.POINTER(vp)]
    L.orbfe_kfdb_destroy.argtypes = [vp]
    L.orbfe_kfdb_destroy.restype = None
    L.orbfe_kfdb_add.argtypes = [vp, i, i, vp, vp]
    L.orbfe_kfdb_add_device.argtypes = [vp, i, vp, vp, i, vp, vp, vp, vp]
    L.orbfe_kfdb_erase.argtypes = [vp, i]
    L.orbfe_kfdb_clear.argtypes = [vp]
    L.orbfe_kfdb_set_covisibles.argtypes = [vp, i, vp, vp, vp]
    L.orbfe_kfdb_size.argtypes = [vp, vp, vp]
    L.orbfe_kfdb_detect.argtypes = [vp, i, i, vp, vp, i, vp, C.c_float, i, vp, vp, vp, vp]
    L.orbfe_kfdb_detect_device.argtypes = [vp, i, i, vp, vp, i, vp, C.c_float, i, vp, vp, vp, vp, vp]
    _kfdb_bound = True
    return L


class KeyFrameDatabase:
    """KeyFrameDatabase (reference src/KeyFrameDatabase.cc) resident on the vocabulary's device: keyframes are slots
    0 <= slot < max_keyframes, the inverted file, BowVectors, covisibility lists and the per-keyframe query fields live in
    device memory (include/orbfe_bow.h, orbfe_kfdb_*)."""

    LOOP, RELOC = 0, 1

    def __init__(self, voc: "Vocabulary", max_keyframes, max_postings):
        L = _bind_kfdb()
        h = C.c_void_p()
        _check(L.orbfe_kfdb_create(voc.handle, int(max_keyframes), int(max_postings), C.byref(h)))
        self._h, self.max_keyframes, self._voc = h.value, int(max_keyframes), voc

    @property
    def handle(self):
        return self._h

    def close(self):
        if self._h:
            lib().orbfe_kfdb_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def add(self, slot, ids, vals):
        ids, vals = np.ascontiguousarray(ids, np.int32), np.ascontiguousarray(vals, np.float64)
        _check(_bind_kfdb().orbfe_kfdb_add(self._h, int(slot), len(ids), _p(ids), _p(vals)))

    def add_device(self, slots, frames, cap, d_bow_ids, d_bow_vals, d_bow_n, stream=0):
        """add() of keyframe slots[i] with the BowVector of row frames[i] that bow_vector_device wrote (ints = raw device
        addresses, row f at f*cap), in order i; all or nothing, synchronous."""
        slots, frames = np.ascontiguousarray(slots, np.int32), np.ascontiguousarray(frames, np.int32)
        if len(slots) != len(frames):
            raise ValueError("slots and frames differ in length")
        vp = C.c_void_p
        _check(_bind_kfdb().orbfe_kfdb_add_device(self._h, len(slots), _p(slots), _p(frames), int(cap), vp(d_bow_ids), vp(d_bow_vals),
                                                  vp(d_bow_n), vp(stream)))

    def erase(self, slot):
        _check(_bind_kfdb().orbfe_kfdb_erase(self._h, int(slot)))

    def clear(self):
        _check(_bind_kfdb().orbfe_kfdb_clear(self._h))

    def set_covisibles(self, lists):
        """lists: {slot: [covisible slots, best first]} (at most 10 each)."""
        slots = np.array(sorted(lists), np.int32)
        ptr = np.zeros(len(slots) + 1, np.int32)
        flat = []
        for k, s in enumerate(slots):
            flat += list(lists[int(s)])
            ptr[k + 1] = len(flat)
        flat = np.array(flat if flat else [0], np.int32)
        _check(_bind_kfdb().orbfe_kfdb_set_covisibles(self._h, len(slots), _p(slots), _p(ptr), _p(flat)))

    def size(self):
        n, p = C.c_int(0), C.c_longlong(0)
        _check(_bind_kfdb().orbfe_kfdb_size(self._h, C.byref(n), C.byref(p)))
        return n.value, p.value

    def detect(self, mode, q_ids, q_vals, connected=(), min_score=0.0, cap=None):
        """(candidate slots, words per slot, score per slot); words / scores are -1 where the query touched nothing."""
        q_ids, q_vals = np.ascontiguousarray(q_ids, np.int32), np.ascontiguousarray(q_vals, np.float64)
        conn = np.ascontiguousarray(connected if len(connected) else [0], np.int32)
        cap = self.max_keyframes if cap is None else int(cap)
        cand = np.zeros(max(cap, 1), np.int32)
        words, score = np.zeros(self.max_keyframes, np.int32), np.zeros(self.max_keyframes, np.float32)
        nc = C.c_int(0)
        _check(_bind_kfdb().orbfe_kfdb_detect(self._h, mode, len(q_ids), _p(q_ids), _p(q_vals), len(connected), _p(conn), min_score, cap,
                                              _p(cand), C.byref(nc), _p(words), _p(score)))
        return cand[:nc.value], words, score

    def detect_device(self, mode, nq, d_q_ids, d_q_vals, nconn, d_connected, min_score, cap, d_cand, d_ncand, d_words=0, d_score=0,
                      stream=0):
        """Device-pointer form (ints = raw device addresses); enqueued, not synchronised."""
        vp = C.c_void_p
        _check(_bind_kfdb().orbfe_kfdb_detect_device(self._h, mode, nq, vp(d_q_ids), vp(d_q_vals), nconn, vp(d_connected), min_score, cap,
                                                     vp(d_cand), vp(d_ncand), vp(d_words or None), vp(d_score or None), vp(stream)))
