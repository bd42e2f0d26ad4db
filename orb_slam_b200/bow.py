"""ctypes wrappers of include/orbfe_bow.h: the DBoW2 vocabulary-tree transform (reference
Thirdparty/DBoW2/DBoW2/TemplatedVocabulary.h:1126-1262; callers Frame.cc:280-287, KeyFrame.cc:56-65) and the batched
MapPoint::ComputeDistinctiveDescriptors and MapPoint::UpdateNormalAndDepth (reference src/MapPoint.cc:185-250, 273-312).
No CPU fallback: every call runs the
CUDA kernels of liborbfe.so."""
import ctypes as C
import os

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
    L.orbfe_vocabulary_load_text.argtypes = [C.c_int, C.c_char_p, C.POINTER(vp)]
    L.orbfe_vocabulary_info.argtypes = [vp] + [C.POINTER(C.c_int)] * 6
    L.orbfe_vocabulary_export.argtypes = [vp, vp, vp, vp, vp, vp, vp]
    L.orbfe_bow_descend_device.argtypes = [vp, vp, C.c_int, C.c_int, vp, vp, vp]
    L.orbfe_bow_descend.argtypes = [vp, vp, C.c_int, C.c_int, vp, vp]
    L.orbfe_bow_transform.argtypes = [vp, vp, C.c_int, C.c_int, vp, vp, vp, vp, vp, vp, vp]
    L.orbfe_distinctive_descriptors.argtypes = [vp, vp, vp, C.c_int, vp]
    L.orbfe_bow_db_detect.argtypes = [vp, C.c_int, C.c_int, vp, vp, C.c_int, vp, vp, vp, vp, vp, vp, C.c_float, vp, vp, vp, vp]
    L.orbfe_feature_vector_device.argtypes = [vp, C.c_int, vp, vp, vp, C.c_int, vp, vp, vp, vp, vp]
    L.orbfe_bow_vector_device.argtypes = [vp, C.c_int, vp, vp, C.c_int, vp, vp, vp, vp]
    L.orbfe_distinctive_descriptors_device.argtypes = [vp, C.c_int, vp, vp, C.c_int, C.c_int, vp, vp, C.c_int, vp, vp, vp]
    L.orbfe_bow_min_score_device.argtypes = [vp, C.c_int, C.c_int, C.c_int, vp, vp, vp, vp, vp, vp, vp, vp, vp]
    L.orbfe_bow_score.argtypes = [vp, C.c_int, vp, vp, C.c_int, vp, vp, vp]
    L.orbfe_normal_and_depth_device.argtypes = [vp, C.c_int, vp, vp, C.c_int, C.c_int, vp, vp, vp, C.c_int, vp, vp, C.c_float, C.c_int, vp,
                                                vp, vp, vp, vp]
    L.orbfe_normal_and_depth.argtypes = [vp, C.c_int, vp, vp, vp, vp, vp, C.c_float, C.c_int, vp, vp, vp, vp]
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

    @classmethod
    def load_text(cls, path, device=0):
        """TemplatedVocabulary::loadFromTextFile (e.g. ORB-SLAM's Data/ORBvoc.txt) parsed on `device`: the node table is
        built in device memory; header, weighting and norm come from the file.  See include/orbfe_bow.h."""
        L = _bind()
        h = C.c_void_p()
        _check(L.orbfe_vocabulary_load_text(int(device), os.fsencode(path), C.byref(h)))
        self = cls.__new__(cls)
        self._h, self.arrays = h.value, None
        return self

    def info(self):
        """dict(k, L, scoring, weighting, nnodes, nwords); k and scoring are -1 for a vocabulary built from arrays."""
        f = [C.c_int(0) for _ in range(6)]
        _check(_bind().orbfe_vocabulary_info(self._h, *[C.byref(x) for x in f]))
        return dict(zip(("k", "L", "scoring", "weighting", "nnodes", "nwords"), (x.value for x in f)))

    def export(self):
        """The node table in the constructor's layout (node_desc, child_ptr, children, word_id, weight) plus parent."""
        n = self.info()["nnodes"]
        child_ptr = np.zeros(n + 1, np.int32)
        _check(_bind().orbfe_vocabulary_export(self._h, None, _p(child_ptr), None, None, None, None))
        out = {"node_desc": np.zeros((n, 32), np.uint8), "child_ptr": child_ptr, "children": np.zeros(max(int(child_ptr[n]), 1), np.int32),
               "word_id": np.zeros(n, np.int32), "weight": np.zeros(n, np.float64), "parent": np.zeros(n, np.int32)}
        _check(_bind().orbfe_vocabulary_export(self._h, _p(out["node_desc"]), None, _p(out["children"]), _p(out["word_id"]),
                                               _p(out["weight"]), _p(out["parent"])))
        out["children"] = out["children"][:child_ptr[n]]
        return out

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

    def score(self, ids1, vals1, ids2, vals2):
        """ORBVocabulary::score of two BowVectors (word ids ascending): the double L1Scoring::score returns."""
        ids1, vals1 = np.ascontiguousarray(ids1, np.int32), np.ascontiguousarray(vals1, np.float64)
        ids2, vals2 = np.ascontiguousarray(ids2, np.int32), np.ascontiguousarray(vals2, np.float64)
        if len(ids1) != len(vals1) or len(ids2) != len(vals2):
            raise ValueError("ids and values differ in length")
        s = C.c_double(0.0)
        _check(_bind().orbfe_bow_score(self._h, len(ids1), _p(ids1), _p(vals1), len(ids2), _p(ids2), _p(vals2), C.byref(s)))
        return s.value


def min_score_device(voc: "Vocabulary", nqueries, nframes, cap, d_bow_ids, d_bow_vals, d_bow_n, d_query_row, d_cov_ptr, d_cov_row,
                     d_scores, d_min_score, stream=0):
    """LoopClosing::DetectLoop's minScore of `nqueries` keyframes on the BowVector rows bow_vector_device wrote (ints = raw
    device addresses; row f at f*cap): query b is row d_query_row[b], its connected keyframes are rows
    d_cov_row[d_cov_ptr[b]:d_cov_ptr[b+1]] (negative = bad, skipped).  d_scores (0 = not wanted) receives the float64 score of
    every pair, d_min_score[b] the float32 minimum starting at 1, which detect_batch_device takes as it is.  Enqueued, not
    synchronised; see include/orbfe_bow.h."""
    vp = C.c_void_p
    _check(_bind().orbfe_bow_min_score_device(voc.handle, nqueries, nframes, cap, vp(d_bow_ids), vp(d_bow_vals), vp(d_bow_n),
                                              vp(d_query_row), vp(d_cov_ptr), vp(d_cov_row), vp(d_scores or None), vp(d_min_score),
                                              vp(stream)))


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


def normal_and_depth(matcher: ORBmatcher, world, ref_centers, ref_octave, group_ptr, obs_centers, scale_factor, scale_factors,
                     normal=None, min_dist=None, max_dist=None):
    """MapPoint::UpdateNormalAndDepth for every point (reference src/MapPoint.cc:273-312) from host arrays: world / ref_centers
    [npoints, 3], ref_octave [npoints], observer centres obs_centers[group_ptr[g] .. group_ptr[g+1]) [.., 3].  Returns
    (normal [npoints, 3], min_dist, max_dist) as float32; the rows of empty groups are those of `normal` / `min_dist` /
    `max_dist` as passed (zeros when not given)."""
    f = lambda x, n: np.ascontiguousarray(x, np.float32).reshape(n, 3)
    group_ptr = np.ascontiguousarray(group_ptr, np.int32)
    n = len(group_ptr) - 1
    world, ref_centers = f(world, n), f(ref_centers, n)
    obs_centers = f(obs_centers, -1) if len(np.asarray(obs_centers).ravel()) else np.zeros((1, 3), np.float32)
    ref_octave = np.ascontiguousarray(ref_octave, np.int32)
    sf = np.ascontiguousarray(scale_factors, np.float32)
    out_n = np.zeros((max(n, 1), 3), np.float32) if normal is None else np.array(f(normal, n), copy=True)
    out_min = np.zeros(max(n, 1), np.float32) if min_dist is None else np.array(min_dist, np.float32, copy=True)
    out_max = np.zeros(max(n, 1), np.float32) if max_dist is None else np.array(max_dist, np.float32, copy=True)
    _check(_bind().orbfe_normal_and_depth(matcher.handle, n, _p(world), _p(ref_centers), _p(ref_octave), _p(group_ptr), _p(obs_centers),
                                          float(scale_factor), len(sf), _p(sf), _p(out_n), _p(out_min), _p(out_max)))
    return out_n[:n], out_min[:n], out_max[:n]


def normal_and_depth_device(matcher: ORBmatcher, npoints, d_kps, d_counts, nframes, cap, d_centers, d_group_ptr, d_obs, nobs, d_world,
                            d_ref_obs, scale_factor, scale_factors, d_normal, d_min_dist, d_max_dist, stream=0):
    """Device-pointer form (ints = raw device addresses) on the frame store and the observation lists of
    distinctive_descriptors_device; d_centers holds 3 floats per frame row, d_ref_obs one slot per point.  Enqueued, not
    synchronised; see include/orbfe_bow.h."""
    vp = C.c_void_p
    sf = np.ascontiguousarray(scale_factors, np.float32)
    _check(_bind().orbfe_normal_and_depth_device(matcher.handle, npoints, vp(d_kps), vp(d_counts), nframes, cap, vp(d_centers),
                                                 vp(d_group_ptr), vp(d_obs), nobs, vp(d_world), vp(d_ref_obs), float(scale_factor), len(sf),
                                                 _p(sf), vp(d_normal), vp(d_min_dist), vp(d_max_dist), vp(stream)))


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
    L.orbfe_kfdb_create_batched.argtypes = [vp, i, C.c_longlong, i, C.POINTER(vp)]
    L.orbfe_kfdb_detect_batch_device.argtypes = [vp, i, i, i, vp, vp, vp, vp, vp, i, vp, vp, vp, vp, vp]
    L.orbfe_kfdb_set_covisibles_device.argtypes = [vp, i, vp, vp, vp, vp]
    L.orbfe_covis_create.argtypes = [i, i, i, i, C.POINTER(vp)]
    L.orbfe_covis_destroy.argtypes = [vp]
    L.orbfe_covis_destroy.restype = None
    L.orbfe_covis_add.argtypes = [vp, i, vp, vp, vp]
    L.orbfe_covis_update_connections_device.argtypes = [vp, i, vp, vp, vp, i, i, vp, vp, i, i, vp, vp]
    L.orbfe_covis_erase.argtypes = [vp, i]
    L.orbfe_covis_clear.argtypes = [vp]
    L.orbfe_covis_lists_device.argtypes = [vp, i, i, vp, i, vp, vp, vp, vp]
    L.orbfe_covis_sync.argtypes = [vp]
    L.orbfe_covis_observations_device.argtypes = [vp, i, vp, i, vp, vp, i, i, vp, i, vp, vp, vp, vp, vp, vp]
    L.orbfe_covis_keyframe_culling_device.argtypes = [vp, i, vp, vp, vp, i, i, vp, vp, i, i, vp, i, vp, vp, vp, vp, vp, vp, vp, vp,
                                                      vp, vp]
    L.orbfe_covis_local_map_device.argtypes = [vp, i, vp, vp, i, vp, vp, i, i, vp, vp, vp, vp, vp, vp, vp]
    _kfdb_bound = True
    return L


class KeyFrameDatabase:
    """KeyFrameDatabase (reference src/KeyFrameDatabase.cc) resident on the vocabulary's device: keyframes are slots
    0 <= slot < max_keyframes, the inverted file, BowVectors, covisibility lists and the per-keyframe query fields live in
    device memory (include/orbfe_bow.h, orbfe_kfdb_*).  max_queries: the largest batch detect_batch_device takes."""

    LOOP, RELOC = 0, 1

    def __init__(self, voc: "Vocabulary", max_keyframes, max_postings, max_queries=1):
        L = _bind_kfdb()
        h = C.c_void_p()
        _check(L.orbfe_kfdb_create_batched(voc.handle, int(max_keyframes), int(max_postings), int(max_queries), C.byref(h)))
        self._h, self.max_keyframes, self.max_queries, self._voc = h.value, int(max_keyframes), int(max_queries), voc

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

    def set_covisibles_device(self, slots, d_ptr, d_lists, stream=0):
        """set_covisibles() with the lists read on the device (ints = raw device addresses): slot slots[i] gets the first 10
        entries of d_lists[d_ptr[i]:d_ptr[i+1]], a CovisibilityGraph.lists_device(0, ...) export as it is; negative entries
        keep their place and contribute nothing.  Enqueued, not synchronised."""
        slots = np.ascontiguousarray(slots, np.int32)
        vp = C.c_void_p
        _check(_bind_kfdb().orbfe_kfdb_set_covisibles_device(self._h, len(slots), _p(slots), vp(d_ptr or None), vp(d_lists or None),
                                                             vp(stream)))

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

    def detect_batch_device(self, mode, nqueries, qcap, d_q_ids, d_q_vals, d_conn_ptr, d_connected, d_min_score, cap, d_cand, d_ncand,
                            d_words=0, d_score=0, stream=0):
        """nqueries queries of one mode as nqueries consecutive detect_device calls (ints = raw device addresses): query b is
        row b of d_q_ids / d_q_vals (qcap entries each); in loop mode its connected slots are
        d_connected[d_conn_ptr[b]:d_conn_ptr[b+1]] and its minScore d_min_score[b].  Row b of d_cand at b*cap, d_ncand[b],
        rows b of d_words / d_score at b*max_keyframes.  Enqueued, not synchronised."""
        vp = C.c_void_p
        _check(_bind_kfdb().orbfe_kfdb_detect_batch_device(self._h, mode, nqueries, qcap, vp(d_q_ids or None), vp(d_q_vals or None),
                                                           vp(d_conn_ptr or None), vp(d_connected or None), vp(d_min_score or None), cap,
                                                           vp(d_cand or None), vp(d_ncand or None), vp(d_words or None), vp(d_score or None),
                                                           vp(stream)))


class CovisibilityGraph:
    """The covisibility graph of one map resident on `device` (include/orbfe_bow.h, orbfe_covis_*): KeyFrame::UpdateConnections
    for batches of keyframes, the connection half of SetBadFlag, and CSR exports of the lists the loop and relocalisation
    queries read.  A keyframe is a slot (its frame-store row) with a 64-bit order key standing for its KeyFrame*."""

    BEST, CONNECTED = 0, 1

    def __init__(self, max_keyframes, max_connections, max_batch=64, device=0):
        L = _bind_kfdb()
        h = C.c_void_p()
        _check(L.orbfe_covis_create(int(device), int(max_keyframes), int(max_connections), int(max_batch), C.byref(h)))
        self._h, self.max_keyframes, self.max_connections, self.max_batch = h.value, int(max_keyframes), int(max_connections), int(max_batch)

    @property
    def handle(self):
        return self._h

    def close(self):
        if self._h:
            lib().orbfe_covis_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def add(self, slots, ids, keys):
        """new keyframes: slot slots[i], mnId ids[i], order key keys[i]; all or nothing, synchronous"""
        slots, ids = np.ascontiguousarray(slots, np.int32), np.ascontiguousarray(ids, np.int32)
        keys = np.ascontiguousarray(keys, np.uint64)
        if not len(slots) == len(ids) == len(keys):
            raise ValueError("slots, ids and keys differ in length")
        _check(_bind_kfdb().orbfe_covis_add(self._h, len(slots), _p(slots), _p(ids), _p(keys)))

    def update_connections_device(self, slots, d_kf_mp, d_counts, nframes, cap, d_group_ptr, d_obs, npoints, nobs, d_parent=0, stream=0):
        """UpdateConnections of slots[0..n) in order (ints = raw device addresses); enqueued, not synchronised.  Bad input or
        an overflowing weight map rejects the batch unchanged and sync() raises."""
        slots = np.ascontiguousarray(slots, np.int32)
        vp = C.c_void_p
        _check(_bind_kfdb().orbfe_covis_update_connections_device(self._h, len(slots), _p(slots), vp(d_kf_mp or None), vp(d_counts or None),
                                                                  int(nframes), int(cap), vp(d_group_ptr or None), vp(d_obs or None),
                                                                  int(npoints), int(nobs), vp(d_parent or None), vp(stream)))

    def erase(self, slot):
        _check(_bind_kfdb().orbfe_covis_erase(self._h, int(slot)))

    def clear(self):
        _check(_bind_kfdb().orbfe_covis_clear(self._h))

    def lists_device(self, which, slots, nbest, d_ptr, d_list, d_weights=0, stream=0):
        """CSR lists of `slots` (which 0: best covisibles / the ordered list when nbest <= 0; 1: connected keyframes in key
        order) into d_ptr (n+1) / d_list / d_weights; retired keyframes are written as -1.  Enqueued, not synchronised."""
        slots = np.ascontiguousarray(slots, np.int32)
        vp = C.c_void_p
        _check(_bind_kfdb().orbfe_covis_lists_device(self._h, int(which), len(slots), _p(slots), int(nbest), vp(d_ptr or None),
                                                     vp(d_list or None), vp(d_weights or None), vp(stream)))

    @staticmethod
    def observations_scratch_bytes(npoints, nframes, cap, obs_cap):
        """bytes of the d_scratch observations_device takes (ORBFE_COVIS_OBS_SCRATCH_BYTES)"""
        return 4 * (2 * int(npoints) + int(obs_cap))

    def observations_device(self, n, d_points, npoints, d_kf_mp, d_counts, nframes, cap, obs_cap, d_ptr, d_obs, d_nobs, d_scratch,
                            d_ref_slot=0, d_ref_obs=0, stream=0):
        """MapPoint::GetObservations() of the n points d_points[0..n) as the inverse of the live slots' rows (ints = raw device
        addresses): point j's entries s*cap + i in key order are d_obs[d_ptr[j]:d_ptr[j+1]], *d_nobs the total, and with
        d_ref_slot, d_ref_obs[j] = ref*cap + observations[ref] (0 when absent).  Enqueued, not synchronised; an overflow or
        bad input writes d_ptr only (and *d_nobs on overflow) and sync() raises."""
        vp = C.c_void_p
        _check(_bind_kfdb().orbfe_covis_observations_device(self._h, int(n), vp(d_points or None), int(npoints), vp(d_kf_mp or None),
                                                            vp(d_counts or None), int(nframes), int(cap), vp(d_ref_slot or None),
                                                            int(obs_cap), vp(d_ptr or None), vp(d_obs or None), vp(d_nobs or None),
                                                            vp(d_ref_obs or None), vp(d_scratch or None), vp(stream)))

    # verdicts of keyframe_culling_device (ORBFE_CULL_*)
    CULL_KEPT, CULL_SKIP_ID0, CULL_ERASED, CULL_NOT_ERASE, CULL_RETIRED = 0, 1, 2, 3, 4

    @staticmethod
    def cull_scratch_bytes(npoints, nframes, cap, obs_cap):
        """bytes of the d_scratch keyframe_culling_device takes (ORBFE_COVIS_CULL_SCRATCH_BYTES)"""
        return 4 * (6 * int(npoints) + 1 + 2 * int(obs_cap) + 2 * int(nframes) + 8) + int(obs_cap)

    def keyframe_culling_device(self, current_slot, d_kf_mp, d_counts, d_kps, nframes, cap, d_point_bad, d_ref_slot, npoints, not_erase,
                                obs_cap, d_nobs, d_verdict_slot, d_verdict, d_ncand, d_bad_points, d_nbad, d_scratch, d_nmps=0,
                                d_nredundant=0, stream=0):
        """LocalMapping::KeyFrameCulling() for the current keyframe current_slot, with SetBadFlag's map-point half (ints = raw
        device addresses; not_erase = the host list of mbNotErase slots).  Verdict t of d_ncand[0] entries is
        (d_verdict_slot[t], d_verdict[t]) with CULL_* codes; d_point_bad / d_ref_slot / the live rows are updated and
        d_bad_points[0:d_nbad[0]] lists the points made bad, ascending.  obs_cap bounds the observation lists of every point
        of the map (they are all built), not only the listed keyframes' points.  Enqueued, not synchronised; bad input or an
        overflow writes nothing (but d_nobs on overflow) and sync() raises."""
        ne = np.ascontiguousarray(not_erase, np.int32)
        vp = C.c_void_p
        _check(_bind_kfdb().orbfe_covis_keyframe_culling_device(
            self._h, int(current_slot), vp(d_kf_mp or None), vp(d_counts or None), vp(d_kps or None), int(nframes), int(cap),
            vp(d_point_bad or None), vp(d_ref_slot or None), int(npoints), len(ne), _p(ne) if len(ne) else None, int(obs_cap),
            vp(d_nobs or None), vp(d_verdict_slot or None), vp(d_verdict or None), vp(d_ncand or None), vp(d_nmps or None),
            vp(d_nredundant or None), vp(d_bad_points or None), vp(d_nbad or None), vp(d_scratch or None), vp(stream)))

    @staticmethod
    def local_map_scratch_bytes(npoints, nframes):
        """bytes of the d_scratch local_map_device takes (ORBFE_COVIS_LOCAL_MAP_SCRATCH_BYTES)"""
        return 4 * (2 * int(npoints) + 4 * int(nframes) + 5)

    def local_map_device(self, nf, d_frame_mp, d_point_bad, npoints, d_kf_mp, d_counts, nframes, cap, d_local_kf, d_nlocal_kf, d_ref_kf,
                         d_local_points, d_nlocal_points, d_scratch, stream=0):
        """Tracking::UpdateReference() for one frame (ints = raw device addresses): the frame's nf cells d_frame_mp lose
        their bad points; d_local_kf[0:d_nlocal_kf[0]] is mvpLocalKeyFrames as slots, d_ref_kf[0] mpReferenceKF (-1 for
        NULL), d_local_points[0:d_nlocal_points[0]] mvpLocalMapPoints.  Enqueued, not synchronised; bad input writes
        nothing and sync() raises."""
        vp = C.c_void_p
        _check(_bind_kfdb().orbfe_covis_local_map_device(
            self._h, int(nf), vp(d_frame_mp or None), vp(d_point_bad or None), int(npoints), vp(d_kf_mp or None), vp(d_counts or None),
            int(nframes), int(cap), vp(d_local_kf or None), vp(d_nlocal_kf or None), vp(d_ref_kf or None), vp(d_local_points or None),
            vp(d_nlocal_points or None), vp(d_scratch or None), vp(stream)))

    def sync(self):
        """waits for the handle's work; raises on the first device-side error since the last sync"""
        _check(_bind_kfdb().orbfe_covis_sync(self._h))
