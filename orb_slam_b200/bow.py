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
