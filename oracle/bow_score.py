"""ORBVocabulary::score and LoopClosing::DetectLoop's minScore loop (src/LoopClosing.cc:117-131) for the tests of
orbfe_bow_min_score_device / orbfe_bow_score (TEST INFRASTRUCTURE ONLY).

  bow_score, loop_min_score   the oracle's restatement, oracle/orb_oracle_bow_score.c, compiled here into
                              oracle/liborb_oracle_bow_score.so with the flags of oracle/Makefile
  RefVocabularyScore          the reference's own ORBVocabulary::score: oracle/ref_shim/ref_voc_score.cc compiled into
                              oracle/_ref/libref_voc_score.so, linked against libref_orbslam.so (the reference's DBoW2,
                              unmodified), where the reference sources exist; elsewhere the prebuilt library is used as it is"""
import ctypes as C
import os
import subprocess

import numpy as np

from . import ref as R

_HERE = os.path.dirname(os.path.abspath(__file__))
_SO = os.path.join(_HERE, "liborb_oracle_bow_score.so")
_SRC = os.path.join(_HERE, "orb_oracle_bow_score.c")
_REF_SO = os.path.join(R._DIR, "libref_voc_score.so")
_REF_SRC = os.path.join(_HERE, "ref_shim", "ref_voc_score.cc")
_lib = None
_ref_lib = None


def build(force=False):
    """Compile the oracle library, and the reference driver where the reference sources exist (after `make ref`)."""
    if force or not os.path.exists(_SO) or os.path.getmtime(_SO) < os.path.getmtime(_SRC):
        subprocess.check_call(["/usr/bin/gcc", "-O3", "-march=x86-64-v3", "-ffp-contract=off", "-fno-fast-math", "-fPIC", "-Wall",
                               "-std=gnu11", "-shared", _SRC, "-o", _SO, "-lm"])
    root = R.REFERENCE_ROOT
    if os.path.isdir(os.path.join(root, "src")):
        base = R.build()
        if force or not os.path.exists(_REF_SO) or os.path.getmtime(_REF_SO) < max(os.path.getmtime(_REF_SRC), os.path.getmtime(base)):
            subprocess.check_call(["/usr/bin/g++", "-std=c++14", "-O2", "-march=x86-64-v3", "-ffp-contract=off", "-fno-fast-math", "-fPIC",
                                   "-w", "-shared", "-I" + os.path.join(_HERE, "ref_shim"), "-I" + os.path.join(root, "include"),
                                   "-I" + root, _REF_SRC, "-o", _REF_SO, "-L" + R._DIR, "-lref_orbslam", "-Wl,-rpath,$ORIGIN",
                                   "-lpthread"])
    return _SO


def ref_available():
    return os.path.exists(_REF_SO) and R.available()


def lib():
    global _lib
    if _lib is None:
        build()
        L = C.CDLL(_SO)
        vp, i = C.c_void_p, C.c_int
        L.orb_oracle_bow_score.argtypes = [vp, vp, i, vp, vp, i]
        L.orb_oracle_bow_score.restype = C.c_double
        L.orb_oracle_loop_min_score.argtypes = [vp, vp, i, i, vp, vp, vp, vp]
        L.orb_oracle_loop_min_score.restype = C.c_float
        _lib = L
    return _lib


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


def _bow(ids, vals):
    return np.ascontiguousarray(ids, np.int32), np.ascontiguousarray(vals, np.float64)


def bow_score(ids1, vals1, ids2, vals2):
    """L1Scoring::score of two BowVectors (word ids ascending), the double ORBVocabulary::score returns."""
    (i1, v1), (i2, v2) = _bow(ids1, vals1), _bow(ids2, vals2)
    return lib().orb_oracle_bow_score(_p(i1), _p(v1), len(i1), _p(i2), _p(v2), len(i2))


def loop_min_score(q_ids, q_vals, covisibles, bad=None):
    """minScore of LoopClosing::DetectLoop as a numpy float32: covisibles = [(ids, vals), ...] in the order of
    GetVectorCovisibleKeyFrames(), bad[k] true for a keyframe with isBad()."""
    qi, qv = _bow(q_ids, q_vals)
    n = len(covisibles)
    ptr = np.cumsum([0] + [len(c[0]) for c in covisibles]).astype(np.int32)
    ci, cv = _bow(np.concatenate([np.asarray(c[0], np.int32) for c in covisibles] + [np.zeros(1, np.int32)]),
                  np.concatenate([np.asarray(c[1], np.float64) for c in covisibles] + [np.zeros(1)]))
    flags = np.zeros(n + 1, np.uint8)
    if bad is not None:
        flags[:n] = np.asarray(bad, bool)
    return np.float32(lib().orb_oracle_loop_min_score(_p(qi), _p(qv), len(qi), n, _p(ptr), _p(ci), _p(cv), _p(flags)))


class RefVocabularyScore:
    """score() of a reference ORBVocabulary loaded from DBoW2's text format."""

    def __init__(self, vocabulary_text_path):
        global _ref_lib
        if _ref_lib is None:
            if not os.path.exists(_REF_SO):
                build()
            L = C.CDLL(_REF_SO, mode=os.RTLD_NOW | os.RTLD_LOCAL)
            vp, i = C.c_void_p, C.c_int
            L.ref_voc_score_create.argtypes = [C.c_char_p]
            L.ref_voc_score_create.restype = vp
            L.ref_voc_score_free.argtypes = [vp]
            L.ref_voc_score_free.restype = None
            L.ref_voc_score.argtypes = [vp, vp, vp, i, vp, vp, i]
            L.ref_voc_score.restype = C.c_double
            _ref_lib = L
        self.L = _ref_lib
        self.h = self.L.ref_voc_score_create(vocabulary_text_path.encode())
        assert self.h, "loadFromTextFile failed"

    def score(self, ids1, vals1, ids2, vals2):
        (i1, v1), (i2, v2) = _bow(ids1, vals1), _bow(ids2, vals2)
        return self.L.ref_voc_score(self.h, _p(i1), _p(v1), len(i1), _p(i2), _p(v2), len(i2))

    def close(self):
        if self.h:
            self.L.ref_voc_score_free(self.h)
            self.h = None
