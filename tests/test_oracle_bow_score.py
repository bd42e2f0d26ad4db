"""CPU tests of the score oracle (oracle/orb_oracle_bow_score.c orb_oracle_bow_score, orb_oracle_loop_min_score), which the device
score (orbfe_bow_min_score_device, orbfe_bow_score) is tested against: it equals the reference's own ORBVocabulary::score
(DBoW2 compiled unmodified into oracle/_ref, called through oracle/ref_shim/ref_voc_score.cc) bit for bit, and its
minimum equals LoopClosing::DetectLoop's loop (LoopClosing.cc:117-131) restated in Python over that reference score with
float32 narrowing."""
import os

import numpy as np
import pytest

import oracle as O
from oracle import ref as R
from oracle import bow_score as OS
from oracle.kfdb import l1_score

import bow_score_scenes as S

needs_ref = pytest.mark.skipif(not OS.ref_available() and not os.path.isdir(os.path.join(R.REFERENCE_ROOT, "src")),
                               reason="oracle/_ref/libref_voc_score.so not built and the reference sources are absent")
PAIRS = S.hand_made_pairs()


@pytest.fixture(scope="module")
def ref_voc(tmp_path_factory):
    path = str(tmp_path_factory.mktemp("bow_score") / "voc2.txt")
    S.tiny_vocabulary_text(path)
    return OS.RefVocabularyScore(path)


def py_min_score(score, q, covisibles, bad):
    """float minScore = 1; float score = ...; if (score < minScore) minScore = score;"""
    m = np.float32(1)
    for c, isbad in zip(covisibles, bad):
        if isbad:
            continue
        s = np.float32(score(q[0], q[1], c[0], c[1]))
        if s < m:
            m = s
    return m


def min_score_cases():
    rng = np.random.default_rng(11)
    q = S.random_bow(rng, 900)
    cov = [S.overlapping(rng, q, keep, 400) for keep in (0.9, 0.5, 0.2, 0.05, 0.0, 0.7)]
    one = S.bow([2, 9, 11], [.5, .25, .25])
    return [
        ("typical", q, cov, [False] * 6),
        ("bad_mixed_in", q, cov, [False, True, False, True, True, False]),
        ("least_is_bad", q, cov, [False, False, False, False, True, False]),
        ("all_bad", q, cov, [True] * 6),
        ("empty_list", q, [], []),
        ("only_itself", one, [one], [False]),                      # score exactly 1: the minimum stays 1
        ("itself_and_others", q, [q] + cov[:2], [False] * 3),
        ("empty_query", S.bow([], []), cov[:2], [False, False]),   # -0.0 < 1
        ("zero_then_nothing_shared", S.bow([1, 2], [1e-200, 1.0]), [S.bow([1], [1e-200]), S.bow([7], [1.0])], [False, False]),
        ("nothing_shared_then_zero", S.bow([1, 2], [1e-200, 1.0]), [S.bow([7], [1.0]), S.bow([1], [1e-200])], [False, False]),
    ]


@pytest.mark.parametrize("name,v1,v2", PAIRS, ids=[p[0] for p in PAIRS])
def test_score_equals_the_plain_python_walk(name, v1, v2):
    """The C oracle against oracle/kfdb.py's l1_score (Python floats, one rounded operation at a time), as bits."""
    got = OS.bow_score(v1[0], v1[1], v2[0], v2[1])
    assert S.bits64([got])[0] == S.bits64([l1_score(v1[0].tolist(), v1[1].tolist(), v2[0].tolist(), v2[1].tolist())])[0]


def test_scenes_hold_their_facts():
    P = {p[0]: p[1:] for p in PAIRS}
    score = lambda n: OS.bow_score(P[n][0][0], P[n][0][1], P[n][1][0], P[n][1][1])
    minus_zero = S.bits64([-0.0])[0]
    for n in ("disjoint", "first_empty", "second_empty", "both_empty"):
        assert S.bits64([score(n)])[0] == minus_zero, n
    assert score("identical_exact_one") == 1.0
    assert abs(score("identical") - 1.0) < 1e-12
    assert abs(score("shared_first") - 0.1) < 1e-15 and abs(score("shared_last") - 0.2) < 1e-15
    assert not 0.0 <= score("not_normalised") <= 1.0
    # the sum's order shows: the same terms added from the last shared word down round differently
    assert score("order_sensitive") != S.reversed_sum_score(*P["order_sensitive"])
    assert len(np.intersect1d(P["order_sensitive"][0][0], P["order_sensitive"][1][0])) > 500


@needs_ref
@pytest.mark.parametrize("name,v1,v2", PAIRS, ids=[p[0] for p in PAIRS])
def test_score_equals_the_reference_on_hand_made_vectors(ref_voc, name, v1, v2):
    for a, b in ((v1, v2), (v2, v1)):
        assert S.bits64([OS.bow_score(a[0], a[1], b[0], b[1])])[0] == S.bits64([ref_voc.score(a[0], a[1], b[0], b[1])])[0]


@needs_ref
@pytest.mark.parametrize("weighting,norm", [(0, 1), (1, 0), (2, 2)])
def test_score_equals_the_reference_on_transformed_descriptors(ref_voc, weighting, norm):
    """BowVectors of orb_oracle_bow_transform from seeded descriptors along a track of the vocabulary's words (L1-normalised as
    ORB-SLAM's, and two weightings / norms whose values are not)."""
    from orb_slam_b200.synth import random_vocabulary
    voc = random_vocabulary(10, 3, seed=6)
    descs = S.track_descriptors(voc, 8, [700, 900, 1, 650, 0, 1000, 33, 800], seed=3, window=600, step=60)
    bows = [O.bow_transform(voc, d, 0, weighting, norm)[0] for d in descs]
    shared = 0
    for a in bows:
        for b in bows:
            assert S.bits64([OS.bow_score(a[0], a[1], b[0], b[1])])[0] == S.bits64([ref_voc.score(a[0], a[1], b[0], b[1])])[0]
            shared += len(np.intersect1d(a[0], b[0]))
    assert shared > 5000


CASES = min_score_cases()


@pytest.mark.parametrize("name,q,cov,bad", CASES, ids=[c[0] for c in CASES])
def test_min_score_equals_the_loop_over_the_oracle_score(name, q, cov, bad):
    got = OS.loop_min_score(q[0], q[1], cov, bad)
    assert got.dtype == np.float32
    assert S.bits32([got])[0] == S.bits32([py_min_score(OS.bow_score, q, cov, bad)])[0]
    if name in ("all_bad", "empty_list", "only_itself"):
        assert S.bits32([got])[0] == S.bits32([1.0])[0]
    if name == "least_is_bad":
        assert got > OS.loop_min_score(q[0], q[1], cov, [False] * len(cov))
    if name == "empty_query":
        assert S.bits32([got])[0] == S.bits32([-0.0])[0]
    # `score < minScore` keeps the first of two zeros of different sign
    if name == "zero_then_nothing_shared":
        assert S.bits32([got])[0] == S.bits32([0.0])[0]
    if name == "nothing_shared_then_zero":
        assert S.bits32([got])[0] == S.bits32([-0.0])[0]


@needs_ref
@pytest.mark.parametrize("name,q,cov,bad", CASES, ids=[c[0] for c in CASES])
def test_min_score_equals_the_loop_over_the_reference_score(ref_voc, name, q, cov, bad):
    assert S.bits32([OS.loop_min_score(q[0], q[1], cov, bad)])[0] == S.bits32([py_min_score(ref_voc.score, q, cov, bad)])[0]
