"""The reference's own KeyFrameDatabase (src/KeyFrameDatabase.cc, compiled unmodified into oracle/_ref/libref_orbslam.so)
behind the slot interface of orbfe_kfdb_*, for replaying scripted sequences (TEST INFRASTRUCTURE ONLY).

oracle/ref_shim/ref_kfdb.cc is the driver, in oracle/_ref/libref_drivers.so, linked against libref_orbslam.so."""
import ctypes as C

import numpy as np

from . import _cdll
from ._cdll import p as _p

vp, i = C.c_void_p, C.c_int
lib = _cdll.loader("_ref/libref_drivers.so", {
    "ref_kfdb_create": (vp, [C.c_char_p]),
    "ref_kfdb_add": (i, [vp, vp, vp, i]),
    "ref_kfdb_erase": (None, [vp, i]),
    "ref_kfdb_clear": (None, [vp]),
    "ref_kfdb_set_covisibles": (None, [vp, i, vp, i]),
    "ref_kfdb_detect_loop": (i, [vp, vp, vp, i, vp, i, C.c_float, vp, i, vp, vp, vp]),
    "ref_kfdb_detect_reloc": (i, [vp, vp, vp, i, vp, i, vp, vp, vp]),
})


def available():
    return _cdll.ref_available("libref_drivers.so")


class RefKeyFrameDatabase:
    """Every add() is a new reference KeyFrame; a slot names the keyframe last added to it.  detect() returns the candidate
    slots and, per slot, the query fields mnLoopWords / mnRelocWords and mLoopScore / mRelocScore of the keyframe the query
    touched there, -1 where it touched none.  The two arrays have max_keyframes entries (as oracle/kfdb.py's); without
    max_keyframes, one entry per slot up to the highest slot added so far."""

    def __init__(self, vocabulary_text_path, max_keyframes=None):
        self.L = lib()
        self.h = self.L.ref_kfdb_create(vocabulary_text_path.encode())
        assert self.h, "loadFromTextFile failed"
        self.K = max_keyframes
        self.k_of, self.slot_of = {}, {}

    def add(self, slot, ids, vals):
        ids, vals = np.ascontiguousarray(ids, np.int32), np.ascontiguousarray(vals, np.float64)
        k = self.L.ref_kfdb_add(self.h, _p(ids), _p(vals), len(ids))
        self.k_of[slot], self.slot_of[k] = k, slot

    def erase(self, slot):
        if slot in self.k_of:
            self.L.ref_kfdb_erase(self.h, self.k_of.pop(slot))

    def clear(self):
        self.L.ref_kfdb_clear(self.h)
        self.k_of.clear()

    def set_covisibles(self, lists):
        for s, lst in lists.items():
            o = np.ascontiguousarray([self.k_of[x] for x in lst] or [0], np.int32)
            self.L.ref_kfdb_set_covisibles(self.h, self.k_of[s], _p(o), len(lst))

    def detect(self, mode, q_ids, q_vals, connected=(), min_score=0.0):
        qi, qv = np.ascontiguousarray(q_ids, np.int32), np.ascontiguousarray(q_vals, np.float64)
        nk = max(len(self.slot_of), 1)
        out, touched, kw, ks = np.zeros(nk, np.int32), np.zeros(nk, np.int32), np.zeros(nk, np.int32), np.zeros(nk, np.float32)
        if mode == 0:
            cn = np.ascontiguousarray([self.k_of[c] for c in connected] or [0], np.int32)
            n = self.L.ref_kfdb_detect_loop(self.h, _p(qi), _p(qv), len(qi), _p(cn), len(connected), float(min_score), _p(out), len(out),
                                            _p(touched), _p(kw), _p(ks))
        else:
            n = self.L.ref_kfdb_detect_reloc(self.h, _p(qi), _p(qv), len(qi), _p(out), len(out), _p(touched), _p(kw), _p(ks))
        assert n <= len(out)
        K = self.K if self.K is not None else max(self.slot_of.values(), default=-1) + 1
        words, scores = np.full(K, -1, np.int32), np.full(K, -1, np.float32)
        for k in np.flatnonzero(touched[:len(self.slot_of)]):
            s = self.slot_of[int(k)]
            assert self.k_of.get(s) == k, "an erased keyframe was touched"
            words[s], scores[s] = kw[k], ks[k]
        return np.array([self.slot_of[int(k)] for k in out[:n]], np.int32), words, scores
