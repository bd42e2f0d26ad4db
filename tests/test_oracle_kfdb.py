"""CPU tests of the stateful keyframe-database oracle (oracle/kfdb.py): over scripted sequences of add / erase / covisibility
changes / clear / slot reuse / interleaved loop and relocalisation queries, its candidate lists (order included) and the
query fields it reports per slot (mnLoopWords / mnRelocWords, and mLoopScore / mRelocScore bit for bit) equal those of the
reference's own KeyFrameDatabase (src/KeyFrameDatabase.cc, compiled unmodified into oracle/_ref and driven by
oracle/ref_shim/ref_kfdb.cc)."""
import os

import numpy as np
import pytest

import oracle as O
from oracle import ref as R
from oracle import ref_kfdb as RK
from oracle.kfdb import KeyFrameDatabase as OracleDB

import kfdb_scenarios as S

pytestmark = pytest.mark.skipif(not RK.available() and not os.path.isdir(os.path.join(R.REFERENCE_ROOT, "src")),
                                reason="oracle/_ref/libref_drivers.so not built and the reference sources are absent")


def same_outputs(got, want, tag):
    """Query outputs (candidates, words, scores) equal, the scores as int32 bits."""
    assert len(got) == len(want), tag
    for q, ((gc, gw, gs), (wc, ww, ws)) in enumerate(zip(got, want)):
        assert np.array_equal(gc, wc), (tag, q, gc, wc)
        assert np.array_equal(gw, ww), (tag, q, np.flatnonzero(gw != ww)[:10])
        assert np.array_equal(gs.view(np.int32), ws.view(np.int32)), (tag, q, np.flatnonzero(gs.view(np.int32) != ws.view(np.int32))[:10])


def _flat_vocabulary_text(path, nwords=10000):
    """10 4 header, a complete 10-ary tree of depth 4: 10^4 words, enough to own every word id of the scenarios."""
    n_nodes = 1 + 10 + 100 + 1000 + nwords
    with open(path, "w") as f:
        f.write("10 4 0 0\n")
        f.write("\n".join("%d %d %s 1.0" % ((nid - 1) // 10, 1 if nid >= 1111 else 0, " ".join(["0"] * 32)) for nid in range(1, n_nodes)))


@pytest.mark.parametrize("seed", [0, 1, 2, 3, 4, 5])
def test_stateful_oracle_equals_the_reference_database(tmp_path, seed):
    path = str(tmp_path / "flat.txt")
    _flat_vocabulary_text(path)
    ops, K = S.mixed_sequence(seed)
    kinds = [op[0] for op in ops]
    assert {"add", "erase", "clear", "covis", "loop", "reloc"} <= set(kinds)
    want = S.replay(RK.RefKeyFrameDatabase(path, K), ops)
    got = S.replay(OracleDB(K), ops)
    same_outputs(got, want, seed)
    assert sum(len(c) > 0 for c, _, _ in want) > len(want) // 2


def test_stale_reloc_score_changes_the_list(tmp_path):
    """The second relocalisation query reads the mRelocScore the first one left (a keyframe touched but not scored): the
    reference, and the stateful oracle, return keyframe B; the stateless oracle, which counts that score as 0, returns A."""
    path = str(tmp_path / "flat.txt")
    _flat_vocabulary_text(path)
    ops = S.stale_reloc_sequence()
    want = S.replay(RK.RefKeyFrameDatabase(path, 3), ops)
    got = S.replay(OracleDB(3), ops)
    same_outputs(got, want, "stale")
    assert got[1][1][1] == 1 and got[1][2][1] == got[0][2][1] > 0   # B: one shared word, the score query 1 left
    assert [list(c) for c, _, _ in got] == [list(c) for c, _, _ in want] == [[1], [1]]
    adds = [op for op in ops if op[0] == "add"]
    kf_ptr = np.cumsum([0] + [len(op[2]) for op in adds]).astype(np.int32)
    cand, _, _ = O.bow_db_detect(1, ops[-1][1], ops[-1][2], kf_ptr, np.concatenate([op[2] for op in adds]),
                                 np.concatenate([op[3] for op in adds]), np.zeros(3, np.uint8), np.array([0, 1, 2, 2], np.int32),
                                 np.array([1, 0], np.int32), 0.0)
    assert list(cand) == [0]
