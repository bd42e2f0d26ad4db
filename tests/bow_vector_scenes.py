"""Vocabularies and a plain-Python BowVector for the tests of orbfe_bow_vector_device (include/orbfe_bow.h).

py_bow_vector restates transform()'s BowVector (TemplatedVocabulary.h:1126-1172, BowVector.cpp:34-84) from leaf ids with
Python floats, which are IEEE doubles added one at a time: values in feature order, the norm summed in ascending word
order.  It takes any leaf ids, so it also covers inputs the descent never produces (ids outside the vocabulary)."""
import math

import numpy as np

from orb_slam_b200 import bow as B
from orb_slam_b200.synth import random_vocabulary, noisy_copies, random_descriptors

# (weighting, norm) of the four transform variants the tests run: the pairs of test_bow_transform_matches_oracle
MODES = [(B.TF_IDF, B.NORM_L1), (B.TF, B.NORM_NONE), (B.IDF, B.NORM_L2), (B.BINARY, B.NORM_L1)]
# DBoW2 ScoringType whose mustNormalize() gives each norm (ScoringObject.h): L1_NORM, L2_NORM, DOT_PRODUCT (none)
SCORING_OF_NORM = {B.NORM_L1: 0, B.NORM_L2: 1, B.NORM_NONE: 5}


def order_vocabulary(seed=3):
    """A k = 10, L = 3 vocabulary whose word weights span four orders of magnitude (10^-2 .. 2*10^2), a few stopped: sums of
    its values depend on the order they are taken in, so a norm taken in any other order than the reference's rounds
    differently (wider spans let the largest terms swallow the rest, and the L2 norm's square root hides the rest)."""
    voc = random_vocabulary(10, 3, seed=seed)
    rng = np.random.default_rng(seed + 100)
    leaf = voc["word_id"] >= 0
    w = 10.0 ** rng.uniform(-2, 2, int(leaf.sum())) * rng.uniform(1, 2, int(leaf.sum()))
    w[rng.random(len(w)) < 0.02] = 0.0
    voc["weight"] = voc["weight"].copy()
    voc["weight"][leaf] = w
    return voc


def frame_descriptors(voc, n, seed):
    """n descriptors near the vocabulary's words (many features per word), every 50th unrelated."""
    words = voc["node_desc"][voc["word_id"] >= 0]
    rng = np.random.default_rng(seed)
    desc = noisy_copies(words[rng.integers(0, len(words), n)], 0.1, seed + 1)
    desc[::50] = random_descriptors(len(desc[::50]), seed + 2)
    return desc


def raw_word_values(voc, leaf, weighting):
    """(word ids ascending, values) before any division: the map built by addWeight / addIfNotExist."""
    wid, wgt = voc["word_id"], voc["weight"]
    vals = {}
    for l in leaf:
        l = int(l)
        if not (0 <= l < len(wgt)) or not (wgt[l] > 0):
            continue
        w, x = int(wid[l]), float(wgt[l])
        if w not in vals:
            vals[w] = x
        elif weighting in (B.TF_IDF, B.TF):
            vals[w] += x
    ids = sorted(vals)
    return ids, [vals[i] for i in ids]


def sequential_norm(v, norm):
    s = 0.0
    if norm == B.NORM_L1:
        for x in v:
            s += abs(x)
    else:
        for x in v:
            s += x * x
        s = math.sqrt(s)
    return s


def py_bow_vector(voc, leaf, weighting, norm):
    ids, v = raw_word_values(voc, leaf, weighting)
    if norm == B.NORM_NONE:
        if weighting in (B.TF_IDF, B.TF) and v:
            v = [x / len(v) for x in v]
    else:
        s = sequential_norm(v, norm)
        if s > 0:
            v = [x / s for x in v]
    return np.array(ids, np.int32), np.array(v, np.float64)


def pairwise_norm(v, norm):
    """numpy's (pairwise, unrolled) sum of the same terms."""
    v = np.asarray(v, np.float64)
    return float(np.sum(np.abs(v))) if norm == B.NORM_L1 else float(np.sqrt(np.sum(v * v)))
