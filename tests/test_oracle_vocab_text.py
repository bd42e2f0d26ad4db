"""The oracle of orbfe_vocabulary_load_text checked on its own: the reference's loadFromTextFile, read out through
oracle/ref_shim/ref_voc_nodes.cc, gives back exactly the arrays of synth.random_vocabulary that oracle.ref.write_vocabulary_text
wrote (nodes by line, children in line order, words in leaf order, weights bit for bit)."""
import os

import numpy as np
import pytest

from oracle import ref as R
from oracle import voc_text as VT
from orb_slam_b200.synth import random_vocabulary

needs_ref = pytest.mark.skipif(not VT.available() and not os.path.isdir(os.path.join(R.REFERENCE_ROOT, "src")),
                               reason="oracle/_ref/libref_drivers.so not built and the reference sources are absent")


def parents_of(voc):
    cp, ch = voc["child_ptr"], voc["children"]
    parent = np.zeros(len(voc["node_desc"]), np.int32)
    for i in range(len(parent)):
        parent[ch[cp[i]:cp[i + 1]]] = i
    return parent


@needs_ref
@pytest.mark.parametrize("k, L, seed, ragged", [(10, 2, 0, False), (4, 4, 1, False), (5, 4, 2, True), (3, 6, 3, True), (10, 3, 4, True)])
@pytest.mark.parametrize("scoring, weighting", [(0, 0), (1, 2), (5, 3)])
def test_reference_nodes_equal_the_written_arrays(tmp_path, k, L, seed, ragged, scoring, weighting):
    voc = random_vocabulary(k, L, seed=seed, ragged=ragged)
    path = str(tmp_path / "voc.txt")
    R.write_vocabulary_text(voc, path, scoring=scoring, weighting=weighting)
    ref = VT.RefVocabularyNodes(path)
    try:
        info, got = ref.info(), ref.nodes()
    finally:
        ref.close()
    n = len(voc["node_desc"])
    leaf = np.diff(voc["child_ptr"]) == 0
    leaf[0] = False
    assert info == {"k": k, "L": L, "scoring": scoring, "weighting": weighting, "nnodes": n, "nchildren": n - 1,
                    "nwords": int(leaf.sum())}
    assert np.array_equal(got["child_ptr"], voc["child_ptr"])
    assert np.array_equal(got["children"], voc["children"])
    assert np.array_equal(got["parent"], parents_of(voc))
    assert np.array_equal(got["node_desc"][1:], voc["node_desc"][1:])
    assert not got["node_desc"][0].any()
    assert np.array_equal(got["word_id"], np.where(leaf, voc["word_id"], 0))
    assert np.array_equal(got["weight"].view(np.uint64), voc["weight"].view(np.uint64))


def test_text_for_reference_drops_one_final_newline(tmp_path):
    src, dst = tmp_path / "a.txt", tmp_path / "b.txt"
    src.write_bytes(b"10 6 0 0\n0 1 " + b"1 " * 32 + b"2\n\n")
    VT.text_for_reference(str(src), str(dst))
    assert dst.read_bytes() == src.read_bytes()[:-1]
