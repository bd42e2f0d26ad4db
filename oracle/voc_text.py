"""The reference's own TemplatedVocabulary::loadFromTextFile and its m_nodes, for the tests of orbfe_vocabulary_load_text
(TEST INFRASTRUCTURE ONLY).

  RefVocabularyNodes   oracle/ref_shim/ref_voc_nodes.cc compiled into oracle/_ref/libref_voc_nodes.so, linked against
                       libref_orbslam.so (the reference's DBoW2, unmodified), where the reference sources exist; elsewhere the
                       prebuilt library is used as it is
  text_for_reference   the text the reference is given: the same bytes without a final newline (a final newline makes the
                       reference read one more, empty line and create a node from uninitialised values)"""
import ctypes as C
import os
import subprocess

import numpy as np

from . import ref as R

_HERE = os.path.dirname(os.path.abspath(__file__))
_REF_SO = os.path.join(R._DIR, "libref_voc_nodes.so")
_REF_SRC = os.path.join(_HERE, "ref_shim", "ref_voc_nodes.cc")
_lib = None


def build(force=False):
    """Compile the driver where the reference sources exist (after `make ref`)."""
    root = R.REFERENCE_ROOT
    if os.path.isdir(os.path.join(root, "src")):
        base = R.build()
        if force or not os.path.exists(_REF_SO) or os.path.getmtime(_REF_SO) < max(os.path.getmtime(_REF_SRC), os.path.getmtime(base)):
            subprocess.check_call(["/usr/bin/g++", "-std=c++14", "-O2", "-march=x86-64-v3", "-ffp-contract=off", "-fno-fast-math", "-fPIC",
                                   "-w", "-shared", "-I" + os.path.join(_HERE, "ref_shim"), "-I" + os.path.join(root, "include"),
                                   "-I" + root, _REF_SRC, "-o", _REF_SO, "-L" + R._DIR, "-lref_orbslam", "-Wl,-rpath,$ORIGIN",
                                   "-lpthread"])
    return _REF_SO


def available():
    return os.path.exists(_REF_SO) and R.available()


def _load():
    global _lib
    if _lib is None:
        if not os.path.exists(_REF_SO):
            build()
        L = C.CDLL(_REF_SO, mode=os.RTLD_NOW | os.RTLD_LOCAL)
        vp, ip = C.c_void_p, C.POINTER(C.c_int)
        L.ref_voc_nodes_load.argtypes = [C.c_char_p, C.POINTER(C.c_double)]
        L.ref_voc_nodes_load.restype = vp
        L.ref_voc_nodes_free.argtypes = [vp]
        L.ref_voc_nodes_free.restype = None
        L.ref_voc_nodes_info.argtypes = [vp] + [ip] * 7
        L.ref_voc_nodes_info.restype = None
        L.ref_voc_nodes_export.argtypes = [vp] * 7
        L.ref_voc_nodes_export.restype = None
        _lib = L
    return _lib


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


def text_for_reference(src, dst):
    """Writes the bytes of file `src` to `dst` without one final newline; returns dst."""
    data = open(src, "rb").read()
    if data.endswith(b"\n"):
        data = data[:-1]
    open(dst, "wb").write(data)
    return dst


class RefVocabularyNodes:
    """A reference ORBVocabulary loaded with loadFromTextFile; `seconds` is that call's wall time."""

    def __init__(self, path):
        self.L = _load()
        t = C.c_double(0.0)
        self.h = self.L.ref_voc_nodes_load(os.fsencode(path), C.byref(t))
        assert self.h, "loadFromTextFile failed"
        self.seconds = t.value

    def info(self):
        f = [C.c_int(0) for _ in range(7)]
        self.L.ref_voc_nodes_info(self.h, *[C.byref(x) for x in f])
        return dict(zip(("k", "L", "scoring", "weighting", "nnodes", "nchildren", "nwords"), (x.value for x in f)))

    def nodes(self):
        """m_nodes as arrays: node_desc, child_ptr, children, word_id, weight, parent."""
        i = self.info()
        n = i["nnodes"]
        out = {"node_desc": np.zeros((n, 32), np.uint8), "child_ptr": np.zeros(n + 1, np.int32),
               "children": np.zeros(max(i["nchildren"], 1), np.int32), "word_id": np.zeros(n, np.int32), "weight": np.zeros(n, np.float64),
               "parent": np.zeros(n, np.int32)}
        self.L.ref_voc_nodes_export(self.h, *[_p(out[k]) for k in ("node_desc", "child_ptr", "children", "word_id", "weight", "parent")])
        out["children"] = out["children"][:i["nchildren"]]
        return out

    def close(self):
        if self.h:
            self.L.ref_voc_nodes_free(self.h)
            self.h = None
