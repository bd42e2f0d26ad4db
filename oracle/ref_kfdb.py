"""The reference's own KeyFrameDatabase (src/KeyFrameDatabase.cc, compiled unmodified into oracle/_ref/libref_orbslam.so)
behind the slot interface of orbfe_kfdb_*, for replaying scripted sequences (TEST INFRASTRUCTURE ONLY).

oracle/ref_shim/ref_kfdb.cc is the driver; build() compiles it into oracle/_ref/libref_kfdb.so, linked against
libref_orbslam.so, where the reference sources exist.  Elsewhere the prebuilt library is used as it is."""
import ctypes as C
import os
import subprocess

import numpy as np

from . import ref as R

_HERE = os.path.dirname(os.path.abspath(__file__))
_SO = os.path.join(R._DIR, "libref_kfdb.so")
_SRC = os.path.join(_HERE, "ref_shim", "ref_kfdb.cc")
_lib = None


def build(force=False):
    """Compile the driver with the flags of oracle/Makefile's reference objects (after `make ref`)."""
    root = R.REFERENCE_ROOT
    if not os.path.isdir(os.path.join(root, "src")):
        return _SO
    base = R.build()
    if not force and os.path.exists(_SO) and os.path.getmtime(_SO) >= max(os.path.getmtime(_SRC), os.path.getmtime(base)):
        return _SO
    cmd = ["/usr/bin/g++", "-std=c++14", "-O2", "-march=x86-64-v3", "-ffp-contract=off", "-fno-fast-math", "-fPIC", "-w", "-shared",
           "-I" + os.path.join(_HERE, "ref_shim"), "-I" + os.path.join(root, "include"), "-I" + root, _SRC, "-o", _SO,
           "-L" + R._DIR, "-lref_orbslam", "-Wl,-rpath,$ORIGIN", "-lpthread"]
    subprocess.check_call(cmd)
    return _SO


def available():
    return os.path.exists(_SO) and os.path.exists(os.path.join(R._DIR, "libref_orbslam.so"))


def lib():
    global _lib
    if _lib is None:
        if not os.path.exists(_SO):
            build()
        L = C.CDLL(_SO, mode=os.RTLD_NOW | os.RTLD_LOCAL)
        vp, i = C.c_void_p, C.c_int
        L.ref_kfdb_create.argtypes = [C.c_char_p]
        L.ref_kfdb_create.restype = vp
        L.ref_kfdb_add.argtypes = [vp, vp, vp, i]
        L.ref_kfdb_erase.argtypes = [vp, i]
        L.ref_kfdb_erase.restype = None
        L.ref_kfdb_clear.argtypes = [vp]
        L.ref_kfdb_clear.restype = None
        L.ref_kfdb_set_covisibles.argtypes = [vp, i, vp, i]
        L.ref_kfdb_set_covisibles.restype = None
        L.ref_kfdb_detect_loop.argtypes = [vp, vp, vp, i, vp, i, C.c_float, vp, i]
        L.ref_kfdb_detect_reloc.argtypes = [vp, vp, vp, i, vp, i]
        _lib = L
    return _lib


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


class RefKeyFrameDatabase:
    """Every add() is a new reference KeyFrame; a slot names the keyframe last added to it.  detect() returns the candidate
    slots (the reference's query fields are not read back: (cands, None, None))."""

    def __init__(self, vocabulary_text_path):
        self.L = lib()
        self.h = self.L.ref_kfdb_create(vocabulary_text_path.encode())
        assert self.h, "loadFromTextFile failed"
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
        out = np.zeros(max(len(self.slot_of), 1), np.int32)
        if mode == 0:
            cn = np.ascontiguousarray([self.k_of[c] for c in connected] or [0], np.int32)
            n = self.L.ref_kfdb_detect_loop(self.h, _p(qi), _p(qv), len(qi), _p(cn), len(connected), float(min_score), _p(out), len(out))
        else:
            n = self.L.ref_kfdb_detect_reloc(self.h, _p(qi), _p(qv), len(qi), _p(out), len(out))
        assert n <= len(out)
        return np.array([self.slot_of[int(k)] for k in out[:n]], np.int32), None, None
