"""GPU tests of ORBVocabulary::score and LoopClosing::DetectLoop's minScore on the device (include/orbfe_bow.h
orbfe_bow_min_score_device, orbfe_bow_score).  Scores are compared as raw float64 bits and minima as raw float32 bits with
the oracle (oracle/orb_oracle_bow_score.c orb_oracle_bow_score / orb_oracle_loop_min_score, pinned to the reference's DBoW2 in
tests/test_oracle_bow_score.py); scenes come from tests/bow_score_scenes.py.  Out-of-range row indices and counts below are
inputs the kernel is specified to skip or clamp."""
import threading

import numpy as np
import pytest

from oracle import bow_score as OS
import orb_slam_b200 as fe
from orb_slam_b200 import bow as B
from orb_slam_b200.synth import random_vocabulary
from oracle.kfdb import F32, KeyFrameDatabase as OracleDB

import bow_score_scenes as S

pytestmark = pytest.mark.gpu

INT32_MAX, INT32_MIN = 2 ** 31 - 1, -2 ** 31
MAX_CAP = 16384   # ORBFE_FV_MAX_CAP


def _torch():
    import torch
    return torch, torch.device("cuda", 0)


def _t(a, dtype=None):
    torch, dev = _torch()
    return torch.from_numpy(np.ascontiguousarray(a, dtype)).to(dev)


@pytest.fixture(scope="module")
def voc():
    return random_vocabulary(10, 4, seed=14)


@pytest.fixture(scope="module")
def V(gpu_required, voc):
    v = B.Vocabulary(voc)
    yield v
    v.close()


def min_score(V, d_store, nframes, cap, query_row, cov_ptr, cov_row, want_scores=True, stream=None):
    """orbfe_bow_min_score_device on a store already on the device (d_ids, d_vals, d_n); d_scores starts as POISON and
    d_min_score as NaN, so every entry the kernel must write, and none it must not, is checked.  Returns (score bits, minima)."""
    torch, dev = _torch()
    d_q, d_p, d_r = _t(query_row, np.int32), _t(cov_ptr, np.int32), _t(cov_row, np.int32)
    d_sc = _t(np.full(max(int(cov_ptr[-1]), 1), S.POISON, np.uint64).view(np.float64))
    d_min = torch.full((len(query_row),), float("nan"), dtype=torch.float32, device=dev)
    torch.cuda.synchronize()
    B.min_score_device(V, len(query_row), nframes, cap, d_store[0].data_ptr(), d_store[1].data_ptr(), d_store[2].data_ptr(),
                       d_q.data_ptr(), d_p.data_ptr(), d_r.data_ptr(), d_sc.data_ptr() if want_scores else 0, d_min.data_ptr(),
                       stream.cuda_stream if stream is not None else 0)
    torch.cuda.synchronize()
    return d_sc.cpu().numpy().view(np.uint64), d_min.cpu().numpy()


def check(V, store, query_row, cov_ptr, cov_row, tag, nframes=None, d_store=None):
    """Device scores and minima of `store` (numpy ids, vals, n) against the oracle; returns (score bits, minima)."""
    F = len(store[2]) if nframes is None else nframes
    cap = store[0].shape[1]
    if d_store is None:
        d_store = (_t(store[0]), _t(store[1]), _t(store[2]))
    want_sc, want_min = S.expected(store, query_row, cov_ptr, cov_row, F)
    got_sc, got_min = min_score(V, d_store, F, cap, query_row, cov_ptr, cov_row)
    assert np.array_equal(got_sc, want_sc), (tag, np.flatnonzero(got_sc != want_sc)[:10])
    assert np.array_equal(S.bits32(got_min), S.bits32(want_min)), (tag, got_min, want_min)
    return got_sc, got_min


def device_store(V, descs, cap, stream=0):
    """Frames of descriptors through descend_device and bow_vector_device, nothing synchronised: (d_ids, d_vals, d_n)."""
    torch, dev = _torch()
    F = len(descs)
    block = np.zeros((F, cap, 32), np.uint8)
    for f, d in enumerate(descs):
        block[f, :len(d)] = d
    d_desc, d_cnt = _t(block), _t(np.array([len(d) for d in descs], np.int32))
    d_leaf, d_node = torch.zeros(F * cap, dtype=torch.int32, device=dev), torch.zeros(F * cap, dtype=torch.int32, device=dev)
    d_ids = torch.full((F, cap), -7, dtype=torch.int32, device=dev)
    d_vals = torch.full((F, cap), float("nan"), dtype=torch.float64, device=dev)
    d_n = torch.full((F,), -7, dtype=torch.int32, device=dev)
    torch.cuda.synchronize()
    V.descend_device(d_desc.data_ptr(), F * cap, 0, d_leaf.data_ptr(), d_node.data_ptr(), stream)
    B.bow_vector_device(V, F, d_leaf.data_ptr(), d_cnt.data_ptr(), cap, d_ids.data_ptr(), d_vals.data_ptr(), d_n.data_ptr(), stream)
    return d_ids, d_vals, d_n


def host_store(d_store):
    _torch()[0].cuda.synchronize()
    return tuple(x.cpu().numpy() for x in d_store)


@pytest.fixture(scope="module")
def track(V, voc):
    """110 frames of 200 .. 1024 extracted-like descriptors along the vocabulary (one empty, one full), as BowVector rows
    built on the device."""
    cap, F = 1024, 110
    rng = np.random.default_rng(21)
    per = rng.integers(200, cap, F)
    per[7], per[8], per[9] = 0, cap, 1
    d_store = device_store(V, S.track_descriptors(voc, F, per, seed=40, step=12), cap)
    store = host_store(d_store)
    assert store[2][7] == 0 and store[2][9] == 1 and store[2].max() > 700
    return d_store, store, cap, F


# ---- the DetectLoop shape ---------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("nqueries", [1, 7, 64])
def test_scores_and_minimum_equal_the_oracle(V, track, nqueries):
    """1, 7 and 64 keyframes with 0 .. 100 connected keyframes each on rows orbfe_bow_vector_device built: bad entries mixed in,
    lists of different queries overlapping, keyframes that are their own covisible (score 1, minimum unchanged)."""
    d_store, store, cap, F = track
    gen = max(nqueries, 2)
    query_row, cov_ptr, cov_row = S.covisibility_lists(nqueries, gen, F)
    lo = gen - nqueries                 # a single query is the second of the scene: 100 entries of every kind
    got_sc, got_min = check(V, store, query_row[lo:], cov_ptr[lo:], cov_row, nqueries, d_store=d_store)
    ks = np.arange(cov_ptr[lo], cov_ptr[-1])
    sc, live = got_sc.view(np.float64)[ks], cov_row[ks] >= 0
    assert (~live).sum() > 3 and (sc[live] > 0.05).sum() > 10 and (sc[live] < 0.9).sum() > 10
    assert (got_min < 1).sum() >= nqueries * 3 // 4 and (got_min > 0).sum() >= nqueries // 2 and got_min[1 - lo] < 1
    own = [k for b in range(lo, gen) for k in range(cov_ptr[b], cov_ptr[b + 1]) if cov_row[k] == query_row[b]]
    assert own and all(abs(got_sc.view(np.float64)[k] - 1.0) < 1e-12 or store[2][cov_row[k]] == 0 for k in own)


def test_a_keyframe_alone_with_itself_keeps_one(V):
    """Values that sum to exactly 1: score(v, v) = 1.0, which is not < 1, so the minimum is the untouched 1.0f."""
    store = S.padded_store([S.bow([2, 9, 11], [.5, .25, .25])], 8)
    sc, mn = check(V, store, [0], [0, 3], [0, -1, 0], "itself")
    assert sc[0] == sc[2] == S.bits64([1.0])[0] and S.bits32(mn)[0] == S.bits32([1.0])[0]


def test_first_of_two_zero_minima_wins(V):
    """`score < minScore` keeps the first of a +0.0f (a score below float range) and a -0.0f (nothing shared) in list order,
    whichever warp scored them."""
    q, tiny, none = S.bow([1, 2], [1e-200, 1.0]), S.bow([1], [1e-200]), S.bow([7], [1.0])
    store = S.padded_store([q, tiny, none], 4)
    _, mn = check(V, store, [0, 0], [0, 2, 4], [1, 2, 2, 1], "zeros")
    assert list(S.bits32(mn)) == list(S.bits32([0.0, -0.0]))


# ---- boundaries -----------------------------------------------------------------------------------------------------------------
def test_shared_words_at_chunk_edges(V):
    """A connected row of 100 words read in chunks of 32 lanes, against queries that share exactly the words at lane 0, lane
    31, both sides of a chunk boundary, the last (partial) chunk, every word, and none (-0.0)."""
    rng = np.random.default_rng(3)
    ids = np.arange(100, dtype=np.int32) * 7 + 3
    vals = rng.uniform(0.1, 1.0, 100) * 10.0 ** rng.uniform(-8, 0, 100)
    row = (ids, vals)
    picks = {"lane0": [0], "lane31": [31], "boundary": [31, 32], "second_boundary": [63, 64], "tail": [96, 99], "edges": [0, 31, 32, 63, 64, 95, 96, 99],
             "all": list(range(100)), "none": []}
    bows = [row]
    for name, pos in picks.items():
        own = np.arange(40, dtype=np.int32) * 7 + 4                # words the row does not have, interleaved with its own
        qi = np.unique(np.concatenate([ids[pos], own])).astype(np.int32)
        bows.append((qi, rng.uniform(0.1, 1.0, len(qi)) * 10.0 ** rng.uniform(-8, 0, len(qi))))
    store = S.padded_store(bows, 160)
    nq = len(picks)
    q = np.arange(1, nq + 1, dtype=np.int32)
    sc, mn = check(V, store, q, np.arange(nq + 1, dtype=np.int32), np.zeros(nq, np.int32), "edges")
    assert sc[-1] == S.bits64([-0.0])[0] and S.bits32(mn)[-1] == S.bits32([-0.0])[0]
    assert len(set(sc.tolist())) == nq
    # and with the roles exchanged: the 100-word row is the query, staged in shared memory
    check(V, store, np.zeros(1, np.int32), np.array([0, nq], np.int32), q, "edges_swapped")


def test_row_lengths_around_a_warp(V):
    """Rows of 0, 1, 31, 32, 33, 64 and 65 words, every row against every row."""
    rng = np.random.default_rng(8)
    base = S.random_bow(rng, 65, nwords=90, decades=6)
    lens = [0, 1, 31, 32, 33, 64, 65]
    bows = [(base[0][:n], base[1][:n] * rng.uniform(0.5, 2.0, n)) for n in lens]
    store = S.padded_store(bows, 65)          # the longest row has d_bow_n == cap
    F = len(lens)
    q = np.arange(F, dtype=np.int32)
    check(V, store, q, np.arange(F + 1, dtype=np.int32) * F, np.tile(q, F), "lengths")


def test_counts_are_clamped_and_tails_never_read(V):
    """d_bow_n negative (an empty row) and above cap (cap words); whatever lies past a row's count (the usual padding, or words
    that would be shared) changes nothing."""
    rng = np.random.default_rng(12)
    cap = 48
    a = S.random_bow(rng, cap, nwords=80)
    bows = [a, S.overlapping(rng, a, 0.6, 5, nwords=80), S.overlapping(rng, a, 0.4, 9, nwords=80), (a[0][:20], a[1][:20])]
    bows = [(i[:cap], v[:cap]) for i, v in bows]
    counts = [cap + 1000, len(bows[1][0]), -4, 20]
    q, p, r = np.array([0, 1, 2, 3], np.int32), np.array([0, 4, 8, 12, 16], np.int32), np.tile(np.arange(4, dtype=np.int32), 4)
    outs = []
    for tail in (None, (int(a[0][-1]), 0.5), (5, float("nan"))):
        outs.append(check(V, S.padded_store(bows, cap, counts, tail), q, p, r, ("clamp", tail)))
    for sc, mn in outs[1:]:
        assert np.array_equal(sc, outs[0][0]) and np.array_equal(S.bits32(mn), S.bits32(outs[0][1]))
    minus_zero = S.bits64([-0.0])[0]
    assert (outs[0][0][8:12] == minus_zero).all() and (outs[0][0][2::4] == minus_zero).all()   # row 2 is empty either way


def test_rows_outside_the_store_are_never_followed(V):
    """Row indices < 0 or >= nframes: skipped as connected keyframes, an empty BowVector as the query.  The store sits between
    guard rows (one before, two after; ids, values and counts) whose contents differ between two runs: the outputs do not."""
    torch, dev = _torch()
    rng = np.random.default_rng(17)
    cap, F = 64, 5
    a = S.random_bow(rng, 50, nwords=200)
    bows = [a] + [S.overlapping(rng, a, 0.5, 10, nwords=200) for _ in range(F - 1)]
    bows = [(i[:cap], v[:cap]) for i, v in bows]
    store = S.padded_store(bows, cap)
    query_row = np.array([0, F, -1, INT32_MAX, 3], np.int32)
    cov = [[1, F, 2, -1, F + 1, INT32_MAX, INT32_MIN, 3], [0, 1], [2], [F, -1], [F + 1, F]]
    cov_ptr = np.cumsum([0] + [len(c) for c in cov]).astype(np.int32)
    cov_row = np.concatenate(cov).astype(np.int32)
    want_sc, want_min = S.expected(store, query_row, cov_ptr, cov_row)
    assert S.bits32(want_min)[3] == S.bits32(want_min)[4] == S.bits32([1.0])[0] and S.bits32(want_min)[1] == S.bits32([-0.0])[0]
    for guard_bow, guard_n in ((a, 50), ((np.full(50, 7, np.int32), np.full(50, float("nan"))), cap)):
        g = S.padded_store([guard_bow] + bows + [guard_bow, guard_bow], cap, [guard_n] + store[2].tolist() + [guard_n, guard_n])
        d_ids, d_vals, d_n = _t(g[0]), _t(g[1]), _t(g[2])
        inner = (d_ids[1:], d_vals[1:], d_n[1:])
        got_sc, got_min = min_score(V, inner, F, cap, query_row, cov_ptr, cov_row)
        assert np.array_equal(got_sc, want_sc) and np.array_equal(S.bits32(got_min), S.bits32(want_min))


def test_scores_may_be_null(V, track):
    d_store, store, cap, F = track
    query_row, cov_ptr, cov_row = S.covisibility_lists(5, 9, F, max_cov=40)
    _, want = S.expected(store, query_row, cov_ptr, cov_row)
    sc, mn = min_score(V, d_store, F, cap, query_row, cov_ptr, cov_row, want_scores=False)
    assert (sc == S.POISON).all() and np.array_equal(S.bits32(mn), S.bits32(want))


def test_largest_rows(V):
    """cap = ORBFE_FV_MAX_CAP with full rows (192 KB of the query staged in shared memory); one more is
    ORBFE_ERR_UNSUPPORTED."""
    torch, dev = _torch()
    rng = np.random.default_rng(23)
    a = S.random_bow(rng, MAX_CAP, nwords=40000, decades=6)
    bows = [a, S.random_bow(rng, MAX_CAP, nwords=40000, decades=6), S.random_bow(rng, MAX_CAP - 1, nwords=40000), S.random_bow(rng, 33, nwords=40000)]
    store = S.padded_store(bows, MAX_CAP)
    q = np.array([0, 1, 3], np.int32)
    sc, _ = check(V, store, q, np.array([0, 4, 8, 12], np.int32), np.tile(np.arange(4, dtype=np.int32), 3), "max_cap")
    assert len(np.intersect1d(bows[0][0], bows[1][0])) > 5000
    z = torch.zeros(8, dtype=torch.float64, device=dev)
    with pytest.raises(fe.OrbfeError) as e:
        B.min_score_device(V, 1, 1, MAX_CAP + 1, *([z.data_ptr()] * 8))
    assert e.value.code == fe.ORBFE_ERR_UNSUPPORTED


# ---- the host form ----------------------------------------------------------------------------------------------------------------
def test_host_score_equals_the_device_scores_and_the_oracle(V, track):
    d_store, store, cap, F = track
    for name, v1, v2 in S.hand_made_pairs():
        if name == "padding_inside":
            continue                       # not a BowVector a host holds: its ids are not strictly ascending
        for a, b in ((v1, v2), (v2, v1)):
            assert S.bits64([V.score(a[0], a[1], b[0], b[1])])[0] == S.bits64([OS.bow_score(a[0], a[1], b[0], b[1])])[0], name
    query_row, cov_ptr, cov_row = np.array([20], np.int32), np.array([0, 6], np.int32), np.array([19, 21, 20, 7, 9, 60], np.int32)
    sc, _ = min_score(V, d_store, F, cap, query_row, cov_ptr, cov_row)
    q = S.row_of(store, 20)
    for k, r in enumerate(cov_row):
        c = S.row_of(store, int(r))
        assert S.bits64([V.score(q[0], q[1], c[0], c[1])])[0] == sc[k], r


def test_host_score_from_two_threads(V, track):
    """Two threads scoring different pairs on one vocabulary each get their own results (the staging block is taken one call
    at a time)."""
    _, store, _, F = track
    pairs = [[(S.row_of(store, a), S.row_of(store, (a + 1 + t) % F)) for a in range(t, 60, 2)] for t in range(2)]
    want = [[S.bits64([OS.bow_score(a[0], a[1], b[0], b[1])])[0] for a, b in ps] for ps in pairs]
    got = [[], []]

    def work(t):
        for _ in range(3):
            got[t] = [S.bits64([V.score(a[0], a[1], b[0], b[1])])[0] for a, b in pairs[t]]

    th = [threading.Thread(target=work, args=(t,)) for t in range(2)]
    [x.start() for x in th]
    [x.join() for x in th]
    assert got == want and len(set(want[0])) > 20


# ---- with the resident database ---------------------------------------------------------------------------------------------------
def test_scores_equal_the_database_loop_scores(V, track):
    """A loop query of row q on a resident database filled from the same rows: for every slot the query scored,
    float32(d_scores) of the pair (q, slot) is the d_score the database reports, bit for bit."""
    torch, dev = _torch()
    d_store, store, cap, F = track
    slots = np.array([f for f in range(30, 70) if f != 50], np.int32)
    db = B.KeyFrameDatabase(V, F, F * cap)
    db.add_device(slots, slots, cap, d_store[0].data_ptr(), d_store[1].data_ptr(), d_store[2].data_ptr())
    d_cand, d_nc = torch.zeros(F, dtype=torch.int32, device=dev), torch.zeros(1, dtype=torch.int32, device=dev)
    d_words, d_score = torch.zeros(F, dtype=torch.int32, device=dev), torch.zeros(F, dtype=torch.float32, device=dev)
    torch.cuda.synchronize()
    db.detect_device(0, cap, d_store[0][50].data_ptr(), d_store[1][50].data_ptr(), 0, d_nc.data_ptr(), 0.0, F, d_cand.data_ptr(), d_nc.data_ptr(),
                     d_words.data_ptr(), d_score.data_ptr())
    torch.cuda.synchronize()
    words, score = d_words.cpu().numpy(), d_score.cpu().numpy()
    sc, _ = min_score(V, d_store, F, cap, np.array([50], np.int32), np.array([0, len(slots)], np.int32), slots)
    min_common = int(F32(words.max()) * F32(0.8))
    scored = [k for k, s in enumerate(slots) if words[s] > min_common]
    assert len(scored) >= 3
    for k in scored:
        assert S.bits32([sc.view(np.float64)[k]])[0] == S.bits32(score)[slots[k]], slots[k]
    db.close()


@pytest.mark.parametrize("nqueries", [1, 8])
@pytest.mark.parametrize("caller_stream", [True, False], ids=["caller_stream", "vocabulary_stream"])
def test_chain_to_the_batched_loop_query(V, voc, nqueries, caller_stream):
    """descend_device -> bow_vector_device -> min_score_device -> detect_batch_device(mode 0) with d_min_score left on the
    device: the candidates are those of the oracle database queried with the oracle's minimum.  On a caller stream all the
    calls are enqueued back to back and the host synchronises once, after the last; without one, the BowVectors and the minimum
    run on the vocabulary's stream, which is drained before the database (which then enqueues on its own stream) is queried."""
    torch, dev = _torch()
    cap, F, K = 1024, 60, 48
    per = np.random.default_rng(31).integers(500, cap, F)
    descs = S.track_descriptors(voc, F, per, seed=70, window=1200, step=25)
    st = torch.cuda.Stream(device=dev) if caller_stream else None
    sp = st.cuda_stream if caller_stream else 0
    # the database holds frames 0 .. K-1; the queries are the last nqueries frames
    prep = device_store(V, descs, cap)
    store = host_store(prep)
    db, odb = B.KeyFrameDatabase(V, F, F * cap, max_queries=nqueries), OracleDB(F)
    slots = np.arange(K, dtype=np.int32)
    db.add_device(slots, slots, cap, prep[0].data_ptr(), prep[1].data_ptr(), prep[2].data_ptr())
    lists = {k: [j for j in (k - 1, k + 1, k - 2, k + 2, k - 3) if 0 <= j < K] for k in range(K)}
    db.set_covisibles(lists)
    for k in range(K):
        odb.add(k, *S.row_of(store, k))
    odb.set_covisibles(lists)
    qrows = np.arange(F - nqueries, F, dtype=np.int32)
    # connected keyframes: the nearest frames of the database, one far behind (it sets the minimum), and a bad one
    conn = [[int(K - 1 - j) for j in range(3 + b % 4)] + ([-1] if b % 2 else []) + [25 + b] for b in range(nqueries)]
    cov_ptr = np.cumsum([0] + [len(c) for c in conn]).astype(np.int32)
    cov_row = np.concatenate(conn).astype(np.int32)
    conn_slots = [[c for c in cs if c >= 0] for cs in conn]
    conn_ptr = np.cumsum([0] + [len(c) for c in conn_slots]).astype(np.int32)
    d_q, d_cp, d_cr = _t(qrows), _t(cov_ptr), _t(cov_row)
    d_conn_ptr, d_conn = _t(conn_ptr), _t(np.concatenate(conn_slots).astype(np.int32))
    d_min = torch.full((nqueries,), float("nan"), dtype=torch.float32, device=dev)
    d_cand, d_nc = torch.zeros((nqueries, F), dtype=torch.int32, device=dev), torch.zeros(nqueries, dtype=torch.int32, device=dev)
    torch.cuda.synchronize()
    d_store = device_store(V, descs, cap, sp)                                  # enqueued, not synchronised
    B.min_score_device(V, nqueries, F, cap, d_store[0].data_ptr(), d_store[1].data_ptr(), d_store[2].data_ptr(), d_q.data_ptr(),
                       d_cp.data_ptr(), d_cr.data_ptr(), 0, d_min.data_ptr(), sp)
    if not caller_stream:
        torch.cuda.synchronize()
    db.detect_batch_device(0, nqueries, cap, d_store[0][F - nqueries].data_ptr(), d_store[1][F - nqueries].data_ptr(), d_conn_ptr.data_ptr(),
                           d_conn.data_ptr(), d_min.data_ptr(), F, d_cand.data_ptr(), d_nc.data_ptr(), 0, 0, sp)
    torch.cuda.synchronize()
    _, want_min = S.expected(store, qrows, cov_ptr, cov_row)
    assert np.array_equal(S.bits32(d_min.cpu().numpy()), S.bits32(want_min)) and (want_min < 1).all()
    cand, nc = d_cand.cpu().numpy(), d_nc.cpu().numpy()
    total = 0
    for b in range(nqueries):
        want, _, _ = odb.detect(0, *S.row_of(store, int(qrows[b])), connected=conn_slots[b], min_score=want_min[b])
        assert np.array_equal(cand[b, :nc[b]], want), (b, cand[b, :nc[b]], want)
        total += len(want)
    assert total > 0
    db.close()
