"""Scenes for the tests of ORBVocabulary::score and LoopClosing::DetectLoop's minScore (include/orbfe_bow.h
orbfe_bow_min_score_device, orbfe_bow_score; oracle/orb_oracle_bow_score.c orb_oracle_bow_score, orb_oracle_loop_min_score).
Everything is generated from seeds with numpy: BowVectors, padded frame stores in the layout orbfe_bow_vector_device writes,
covisibility lists, and the expected outputs computed with the oracle."""
import numpy as np

from oracle import bow_score as OS
from orb_slam_b200.synth import noisy_copies

INT32_MAX = 2 ** 31 - 1
F32 = np.float32
POISON = 0x7FF8DEADBEEF0001      # a NaN payload: d_scores entries the kernel must leave alone


def bits64(x):
    return np.ascontiguousarray(x, np.float64).view(np.uint64)


def bits32(x):
    return np.ascontiguousarray(x, np.float32).view(np.uint32)


def tiny_vocabulary_text(path):
    """Two words under the root in DBoW2's text format, L1 scoring and TF-IDF weighting (the header of ORBvoc): score() of
    the loaded vocabulary is L1Scoring::score whatever words the vectors name."""
    with open(path, "w") as f:
        f.write("2 1 0 0\n")
        f.write("\n".join("0 1 %s 1.0" % " ".join(["0"] * 32) for _ in range(2)))


def bow(ids, vals):
    return np.asarray(ids, np.int32), np.asarray(vals, np.float64)


def random_bow(rng, n, nwords=100000, normalise=True, decades=0.0):
    """n distinct ascending word ids below nwords; values uniform, or spread over `decades` orders of magnitude so that the
    order of the score's sum shows in its last bits."""
    ids = np.sort(rng.choice(nwords, n, replace=False)).astype(np.int32)
    v = rng.uniform(0.2, 3.0, n) * (10.0 ** rng.uniform(-decades, 0, n) if decades else 1.0)
    return ids, (v / v.sum() if normalise and n else v)


def overlapping(rng, base, keep, extra, nwords=100000, decades=0.0):
    """A BowVector sharing about `keep` of base's words (with its own values) plus `extra` words of its own."""
    ids = base[0][rng.random(len(base[0])) < keep]
    own = rng.choice(nwords, extra, replace=False).astype(np.int32)
    ids = np.unique(np.concatenate([ids, own])).astype(np.int32)
    v = rng.uniform(0.2, 3.0, len(ids)) * (10.0 ** rng.uniform(-decades, 0, len(ids)) if decades else 1.0)
    return ids, v / v.sum()


def hand_made_pairs():
    """(name, v1, v2) for the decision points of L1Scoring::score."""
    rng = np.random.default_rng(5)
    a = random_bow(rng, 40)
    spread = random_bow(rng, 1500, decades=9)
    out = [
        ("disjoint", bow([1, 3, 5], [.2, .3, .5]), bow([0, 2, 4, 6], [.25, .25, .25, .25])),
        ("identical", a, a),
        ("identical_exact_one", bow([2, 9, 11], [.5, .25, .25]), bow([2, 9, 11], [.5, .25, .25])),
        ("first_empty", bow([], []), a),
        ("second_empty", a, bow([], [])),
        ("both_empty", bow([], []), bow([], [])),
        ("shared_first", bow([0, 10, 20, 30], [.1, .2, .3, .4]), bow([0, 11, 21, 31, 41], [.5, .1, .1, .1, .2])),
        ("shared_last", bow([1, 10, 20, 99], [.1, .2, .3, .4]), bow([0, 11, 21, 31, 99], [.5, .1, .1, .1, .2])),
        ("not_normalised", bow([3, 4, 8, 20], [7.5, 1e3, 0.125, 3e-7]), bow([3, 8, 20, 21], [2.5e2, 9.0, 1e-9, 4.0])),
        ("negative_values", bow([3, 4, 8], [-0.5, 0.25, 0.75]), bow([3, 4, 9], [0.5, -0.25, 1.0])),
        ("padding_inside", bow([5, INT32_MAX, INT32_MAX], [1.0, 0.0, 0.0]), bow([5, 7, INT32_MAX], [0.5, 0.5, 0.0])),
        ("order_sensitive", spread, overlapping(rng, spread, 0.7, 300, decades=9)),
    ]
    return out


def reversed_sum_score(v1, v2):
    """The score with the shared words' terms added in descending word order: differs from L1Scoring::score in the last bits
    on order-sensitive vectors."""
    _, i1, i2 = np.intersect1d(v1[0], v2[0], return_indices=True)
    s = 0.0
    for a, b in zip(i1[::-1], i2[::-1]):
        vi, wi = float(v1[1][a]), float(v2[1][b])
        s += abs(vi - wi) - abs(vi) - abs(wi)
    return -s / 2.0


# ---- frame stores ---------------------------------------------------------------------------------------------------------------
def padded_store(bows, cap, counts=None, tail=None):
    """Rows in the layout orbfe_bow_vector_device writes: row f = bows[f], then id INT32_MAX / value 0.0 up to cap.  counts
    replaces d_bow_n (negative or above cap to be clamped); tail = (id, value) replaces the padding, which the score must
    never read past a row's count."""
    F = len(bows)
    ids = np.full((F, cap), INT32_MAX if tail is None else tail[0], np.int32)
    vals = np.full((F, cap), 0.0 if tail is None else tail[1], np.float64)
    n = np.zeros(F, np.int32)
    for f, (i, v) in enumerate(bows):
        ids[f, :len(i)], vals[f, :len(i)], n[f] = i, v, len(i)
    if counts is not None:
        n = np.asarray(counts, np.int32)
    return ids, vals, n


def row_of(store, f, nframes=None):
    """The BowVector the score reads from row f: its first min(max(n, 0), cap) words; empty for a row outside the store."""
    ids, vals, n = store
    if not 0 <= f < (len(n) if nframes is None else nframes):
        return bow([], [])
    c = min(max(int(n[f]), 0), ids.shape[1])
    return ids[f, :c], vals[f, :c]


def expected(store, query_row, cov_ptr, cov_row, nframes=None):
    """(d_scores as uint64 bits with POISON where the kernel writes nothing, d_min_score as float32) from the oracle."""
    F = len(store[2]) if nframes is None else nframes
    scores = np.full(max(int(cov_ptr[-1]), 1), POISON, np.uint64)
    mins = np.zeros(len(query_row), np.float32)
    for b, q in enumerate(query_row):
        qv = row_of(store, int(q), F)
        cov, bad = [], []
        for k in range(int(cov_ptr[b]), int(cov_ptr[b + 1])):
            r = int(cov_row[k])
            ok = 0 <= r < F
            cv = row_of(store, r, F)
            cov.append(cv)
            bad.append(not ok)
            if ok:
                scores[k] = bits64([OS.bow_score(qv[0], qv[1], cv[0], cv[1])])[0]
        mins[b] = OS.loop_min_score(qv[0], qv[1], cov, bad)
    return scores, mins


def track_descriptors(voc, nframes, per_frame, seed, window=1500, step=40):
    """Descriptors of `nframes` frames moving along the vocabulary's words: frame f draws per_frame[f] noisy copies of words
    from a window that advances by `step`, so neighbouring frames share many words and distant ones few."""
    words = voc["node_desc"][voc["word_id"] >= 0]
    rng = np.random.default_rng(seed)
    out = []
    for f in range(nframes):
        pick = (f * step + rng.integers(0, window, per_frame[f])) % len(words)
        out.append(noisy_copies(words[pick], 0.05, seed + 1 + f))
    return out


def covisibility_lists(seed, nqueries, nframes, max_cov=100, bad_fraction=0.15):
    """query_row, cov_ptr, cov_row for `nqueries` keyframes: 0 .. max_cov connected keyframes each (the first query has none,
    the second every kind), nearest neighbours first with frames up to 25 away mixed in, some bad (-1), lists of different
    queries overlapping, and every third query its own covisible."""
    rng = np.random.default_rng(seed)
    query_row = rng.integers(0, nframes, nqueries).astype(np.int32)
    ptr, rows = [0], []
    for b in range(nqueries):
        ncov = 0 if b == 0 else max_cov if b == 1 else int(rng.integers(0, max_cov + 1))
        near = (query_row[b] + np.array([(-1) ** j * (j // 2 + 1) for j in range(ncov)])) % nframes
        far = (query_row[b] + rng.integers(-25, 26, ncov)) % nframes
        lst = np.where(rng.random(ncov) < 0.7, near, far).astype(np.int32)
        lst[rng.random(ncov) < bad_fraction] = -1
        if b % 3 == 1 and ncov:
            lst[ncov // 2] = query_row[b]
        rows += lst.tolist()
        ptr.append(len(rows))
    return query_row, np.array(ptr, np.int32), np.array(rows if rows else [0], np.int32)
