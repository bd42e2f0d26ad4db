"""The reference's own TemplatedVocabulary::loadFromTextFile and its m_nodes, for the tests of orbfe_vocabulary_load_text
(TEST INFRASTRUCTURE ONLY).

  RefVocabularyNodes   oracle/ref_shim/ref_voc_nodes.cc in oracle/_ref/libref_drivers.so, linked against libref_orbslam.so
                       (the reference's DBoW2, unmodified)
  text_for_reference   the text the reference is given: the same bytes without a final newline (a final newline makes the
                       reference read one more, empty line and create a node from uninitialised values)"""
import ctypes as C
import os

import numpy as np

from . import _cdll
from ._cdll import p as _p

_load = _cdll.loader("_ref/libref_drivers.so", {
    "ref_voc_nodes_load": (C.c_void_p, [C.c_char_p, C.POINTER(C.c_double)]),
    "ref_voc_nodes_free": (None, [C.c_void_p]),
    "ref_voc_nodes_info": (None, [C.c_void_p] + [C.POINTER(C.c_int)] * 7),
    "ref_voc_nodes_export": (None, [C.c_void_p] * 7),
})


def available():
    return _cdll.ref_available("libref_drivers.so")


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
