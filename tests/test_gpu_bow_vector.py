"""GPU tests of the device BowVector (include/orbfe_bow.h orbfe_bow_vector_device) and of the keyframe database fed from it
(orbfe_kfdb_add_device, orbfe_kfdb_detect_device on a padded row).  BowVector values are compared as raw float64 bits
with orbfe_bow_transform, the oracle and a plain-Python restatement (tests/bow_vector_scenes.py); database results
(candidates in order, shared-word counts, float scores bit for bit) with a twin database built by host adds and with the
stateful oracle (oracle/kfdb.py)."""
import numpy as np
import pytest

import oracle as O
import orb_slam_b200 as fe
from orb_slam_b200 import bow as B
from orb_slam_b200.synth import random_vocabulary
from oracle.kfdb import KeyFrameDatabase as OracleDB

import bow_vector_scenes as S
import kfdb_scenarios as KS

pytestmark = pytest.mark.gpu

INT32_MAX = 2 ** 31 - 1
MAX_CAP = 16384   # ORBFE_FV_MAX_CAP


def _torch():
    import torch
    return torch, torch.device("cuda", 0)


def _t(a):
    torch, dev = _torch()
    return torch.from_numpy(np.ascontiguousarray(a)).to(dev)


def flat_vocabulary(nwords):
    """A root with nwords leaf children: a vocabulary that only has to own the word ids 0 .. nwords-1."""
    n = nwords + 1
    child_ptr = np.zeros(n + 1, np.int32)
    child_ptr[1:] = nwords
    return {"node_desc": np.zeros((n, 32), np.uint8), "child_ptr": child_ptr, "children": np.arange(1, n, dtype=np.int32),
            "word_id": np.arange(-1, nwords, dtype=np.int32), "weight": np.ones(n), "L": 1}


def device_bow(V, leaf_rows, counts, cap):
    """orbfe_bow_vector_device on leaf ids uploaded as frames of `cap` entries; outputs start poisoned, so every entry the
    kernel must write is checked.  Returns (ids, vals, n) as numpy arrays."""
    torch, dev = _torch()
    F = len(counts)
    d_leaf, d_cnt = _t(np.asarray(leaf_rows, np.int32).reshape(F * cap)), _t(np.asarray(counts, np.int32))
    d_ids = torch.full((F, cap), -7, dtype=torch.int32, device=dev)
    d_vals = torch.full((F, cap), float("nan"), dtype=torch.float64, device=dev)
    d_n = torch.full((F,), -7, dtype=torch.int32, device=dev)
    s = torch.cuda.Stream(device=dev)
    torch.cuda.synchronize()
    B.bow_vector_device(V, F, d_leaf.data_ptr(), d_cnt.data_ptr(), cap, d_ids.data_ptr(), d_vals.data_ptr(), d_n.data_ptr(), s.cuda_stream)
    s.synchronize()
    return d_ids.cpu().numpy(), d_vals.cpu().numpy(), d_n.cpu().numpy()


def check_row(ids, vals, n, want_ids, want_vals, tag):
    want_vals = np.ascontiguousarray(want_vals, np.float64)
    assert n == len(want_ids), (tag, n, len(want_ids))
    assert np.array_equal(ids[:n], want_ids), tag
    assert np.array_equal(np.ascontiguousarray(vals[:n]).view(np.uint64), want_vals.view(np.uint64)), tag
    assert (ids[n:] == INT32_MAX).all() and (np.ascontiguousarray(vals[n:]).view(np.uint64) == 0).all(), tag   # padding, +0.0


def _same(got, want, tag):
    assert len(got) == len(want), tag
    for q, ((gc, gw, gs), (wc, ww, ws)) in enumerate(zip(got, want)):
        assert np.array_equal(gc, wc), (tag, q, gc, wc)
        assert np.array_equal(gw, ww), (tag, q)
        assert np.array_equal(gs.view(np.int32), ws.view(np.int32)), (tag, q)   # bit for bit


# ---- orbfe_bow_vector_device --------------------------------------------------------------------------------------------
VOCABS = [(10, 4, False), (7, 3, True), (40, 2, False), (10, 5, True), "order"]


@pytest.mark.parametrize("vk", VOCABS, ids=lambda v: v if isinstance(v, str) else "k%d_L%d_%s" % (v[0], v[1], "ragged" if v[2] else "full"))
def test_bow_vector_equals_transform_and_oracle(gpu_required, vk):
    """Frames with 0, 1, a typical number, exactly cap, a negative count and more than cap features in one launch: every row
    equals orbfe_bow_transform and the oracle on the frame's first min(max(count, 0), cap) descriptors, for all four
    (weighting, norm) pairs, on the vocabularies of test_bow_transform_matches_oracle and on the order-discriminating one."""
    voc = S.order_vocabulary() if vk == "order" else random_vocabulary(vk[0], vk[1], seed=vk[0] + vk[1], ragged=vk[2])
    cap = 1024
    counts = [0, 1, 517, cap, -3, cap + 50, 2]
    F = len(counts)
    desc = np.stack([S.frame_descriptors(voc, cap, seed=10 + f) for f in range(F)])
    for weighting, norm in S.MODES:
        V = B.Vocabulary(voc, weighting, norm)
        leaf, _ = V.descend(desc.reshape(F * cap, 32), 0)
        ids, vals, nw = device_bow(V, leaf, counts, cap)
        for f, c in enumerate(counts):
            n = min(max(c, 0), cap)
            (hi, hv), _ = V.transform(desc[f, :n], 0)
            (oi, ov), _ = O.bow_transform(voc, desc[f, :n], 0, weighting, norm)
            check_row(ids[f], vals[f], nw[f], hi, hv, ("transform", f, weighting, norm))
            check_row(ids[f], vals[f], nw[f], oi, ov, ("oracle", f, weighting, norm))
        assert nw[2] > 100 and nw[0] == 0 and nw[4] == 0 and nw[1] == 1
        V.close()


def test_bow_vector_edge_rows(gpu_required):
    """Rows the descent cannot produce, against the plain-Python BowVector: every feature in one word, every word stopped
    (zero-weight leaves and inner nodes), leaf ids outside the vocabulary mixed in, a few heavily repeated words; padding
    on every row."""
    INT32_MIN = -2 ** 31
    for voc in (random_vocabulary(10, 3, seed=4), S.order_vocabulary()):
        nn = len(voc["weight"])
        live = np.flatnonzero((voc["word_id"] >= 0) & (voc["weight"] > 0))
        dead = np.flatnonzero(voc["weight"] == 0)
        cap = 600
        rng = np.random.default_rng(9)
        rows = np.zeros((6, cap), np.int64)
        rows[0] = live[3]
        rows[1] = rng.choice(dead, cap)
        rows[2] = rng.choice(live, cap)
        rows[2, ::3] = rng.choice([-1, INT32_MIN, nn, nn + 5, INT32_MAX], len(rows[2, ::3]))
        rows[3] = rng.choice(live[:5], cap)
        rows[4] = rng.choice(live, cap)
        rows[5] = rng.choice(np.concatenate([live[:50], dead[:20], [-1, nn]]), cap)
        counts = [cap, cap, cap, cap - 1, cap, 333]
        for weighting, norm in S.MODES:
            V = B.Vocabulary(voc, weighting, norm)
            ids, vals, nw = device_bow(V, rows.astype(np.int32), counts, cap)
            for f in range(len(counts)):
                check_row(ids[f], vals[f], nw[f], *S.py_bow_vector(voc, rows[f, :counts[f]], weighting, norm), (f, weighting, norm))
            assert nw[0] == 1 and nw[1] == 0 and nw[3] == 5 and (nw < cap).all()
            V.close()


def test_bow_vector_cap_limit(gpu_required):
    """cap = ORBFE_FV_MAX_CAP is accepted (128 KB of keys in shared memory) and gives the plain-Python BowVector; one more
    is ORBFE_ERR_UNSUPPORTED."""
    torch, dev = _torch()
    voc = S.order_vocabulary()
    live = np.flatnonzero(voc["weight"] > 0)
    rng = np.random.default_rng(2)
    cap = MAX_CAP
    rows = rng.choice(np.concatenate([live, [-1]]), (2, cap)).astype(np.int32)
    counts = [cap, cap - 777]
    for weighting, norm in S.MODES:
        V = B.Vocabulary(voc, weighting, norm)
        ids, vals, nw = device_bow(V, rows, counts, cap)
        for f in range(2):
            check_row(ids[f], vals[f], nw[f], *S.py_bow_vector(voc, rows[f, :counts[f]], weighting, norm), (f, weighting, norm))
        V.close()
    V = B.Vocabulary(voc)
    z = torch.zeros(2 * (cap + 1), dtype=torch.float64, device=dev)
    with pytest.raises(fe.OrbfeError) as e:
        B.bow_vector_device(V, 2, z.data_ptr(), z.data_ptr(), cap + 1, z.data_ptr(), z.data_ptr(), z.data_ptr())
    assert e.value.code == fe.ORBFE_ERR_UNSUPPORTED
    V.close()


# ---- detect_device on a padded row --------------------------------------------------------------------------------------
def _detect_device(db, mode, ids, vals, nq, conn, min_score, K):
    torch, dev = _torch()
    d_qi, d_qv = _t(np.asarray(ids, np.int32)), _t(np.asarray(vals, np.float64))
    conn = np.asarray(conn, np.int32)
    d_conn = _t(conn if len(conn) else np.zeros(1, np.int32))
    d_cand, d_n = torch.zeros(K, dtype=torch.int32, device=dev), torch.zeros(1, dtype=torch.int32, device=dev)
    d_words, d_score = torch.zeros(K, dtype=torch.int32, device=dev), torch.zeros(K, dtype=torch.float32, device=dev)
    torch.cuda.synchronize()
    db.detect_device(mode, nq, d_qi.data_ptr(), d_qv.data_ptr(), len(conn), d_conn.data_ptr(), min_score, K, d_cand.data_ptr(),
                     d_n.data_ptr(), d_words.data_ptr(), d_score.data_ptr())
    torch.cuda.synchronize()
    n = int(d_n.item())
    return d_cand[:n].cpu().numpy(), d_words.cpu().numpy(), d_score.cpu().numpy()


def _replay_detect_device(db, ops, K, pad_to=None):
    out = []
    for op in ops:
        if op[0] in ("loop", "reloc"):
            ids, vals = np.asarray(op[1], np.int32), np.asarray(op[2], np.float64)
            n = len(ids)
            if pad_to is not None:
                ids = np.concatenate([ids, np.full(pad_to - n, INT32_MAX, np.int32)])
                vals = np.concatenate([vals, np.zeros(pad_to - n)])
            mode = 0 if op[0] == "loop" else 1
            out.append(_detect_device(db, mode, ids, vals, len(ids), op[3] if mode == 0 else [], op[4] if mode == 0 else 0.0, K))
        else:
            KS.replay(db, [op])
    return out


@pytest.mark.parametrize("seq", ["stale", 0, 1])
def test_padded_query_equals_unpadded(gpu_required, seq):
    """A query row padded with INT32_MAX / 0.0 up to cap and passed whole gives the candidates, words and scores of its real
    words, query after query: the scores it leaves behind are the ones a later relocalisation reads."""
    V = B.Vocabulary(flat_vocabulary(3000))
    ops, K = (KS.stale_reloc_sequence(), 3) if seq == "stale" else KS.mixed_sequence(seq)
    cap = 1024
    padded, plain = B.KeyFrameDatabase(V, K, 1 << 16), B.KeyFrameDatabase(V, K, 1 << 16)
    got = _replay_detect_device(padded, ops, K, pad_to=cap)
    want = _replay_detect_device(plain, ops, K)
    _same(got, want, seq)
    _same(got, KS.replay(OracleDB(K), ops), seq)
    if seq == "stale":
        assert list(got[1][0]) == [1]   # the score query 1 left in keyframe 1 decides query 2
    padded.close(); plain.close(); V.close()


# ---- orbfe_kfdb_add_device -----------------------------------------------------------------------------------------------
class RowTable:
    """BowVectors as padded device rows (the layout orbfe_bow_vector_device writes): row f = bows[f]; n_override replaces
    the word counts (to build malformed rows)."""

    def __init__(self, bows, cap=None, n_override=None):
        cap = cap or max(1, max(len(b[0]) for b in bows))
        ids = np.full((len(bows), cap), INT32_MAX, np.int32)
        vals = np.zeros((len(bows), cap))
        for f, (i, v) in enumerate(bows):
            ids[f, :len(i)] = i
            vals[f, :len(v)] = v
        n = np.array([len(b[0]) for b in bows] if n_override is None else n_override, np.int32)
        self.cap, self.d_ids, self.d_vals, self.d_n = cap, _t(ids), _t(vals), _t(n)
        _torch()[0].cuda.synchronize()

    def add(self, db, slots, frames):
        db.add_device(slots, frames, self.cap, self.d_ids.data_ptr(), self.d_vals.data_ptr(), self.d_n.data_ptr())


class DeviceAdds:
    """A KeyFrameDatabase whose add() goes through add_device from a RowTable of every BowVector the sequence adds, in order."""

    def __init__(self, db, ops):
        self.db, self.next = db, 0
        self.table = RowTable([(op[2], op[3]) for op in ops if op[0] == "add"])

    def add(self, slot, ids, vals):
        self.table.add(self.db, [slot], [self.next])
        self.next += 1

    def __getattr__(self, name):
        return getattr(self.db, name)


@pytest.mark.parametrize("seed", [0, 1, 2])
def test_add_device_in_mixed_sequences(gpu_required, seed):
    """add_device mixed with erase, covisibility refresh, clear and both queries equals a twin built by host adds and the oracle."""
    V = B.Vocabulary(flat_vocabulary(3000))
    ops, K = KS.mixed_sequence(seed)
    dev_db, host_db = B.KeyFrameDatabase(V, K, 1 << 16), B.KeyFrameDatabase(V, K, 1 << 16)
    got = KS.replay(DeviceAdds(dev_db, ops), ops)
    _same(got, KS.replay(host_db, ops), seed)
    _same(got, KS.replay(OracleDB(K), ops), seed)
    assert dev_db.size() == host_db.size()
    dev_db.close(); host_db.close(); V.close()


def test_batched_add_equals_sequential_adds(gpu_required):
    """One add_device of many keyframes (neighbours share most words, so their links go to the same lists) equals the same
    keyframes added one by one in the same order: same inverted-file order, same candidates, words and scores."""
    V = B.Vocabulary(flat_vocabulary(3000))
    K = 48
    bows, at = KS.trajectory(K, 3000, 120, seed=2)
    slots = np.random.default_rng(5).permutation(K).astype(np.int32)
    table = RowTable(bows)
    batch, seq = B.KeyFrameDatabase(V, K, 1 << 16), B.KeyFrameDatabase(V, K, 1 << 16)
    orc = OracleDB(K)
    table.add(batch, slots[:30], np.arange(30))
    table.add(batch, slots[30:], np.arange(30, K))
    for f in range(K):
        seq.add(int(slots[f]), *bows[f])
        orc.add(int(slots[f]), *bows[f])
    assert batch.size() == seq.size()
    lists = {int(slots[f]): [int(slots[g]) for g in (f - 1, f + 1, f - 2, f + 2) if 0 <= g < K] for f in range(K)}
    for o in (batch, seq, orc):
        o.set_covisibles(lists)
    queries = [at(max(1, 120 // 8) * int(q) + 3, 900 + q) for q in (2, 11, 25, 40, 2)]
    run = lambda o: [o.detect(q % 2, *qb, [int(slots[q])], 0.0) if q % 2 == 0 else o.detect(1, *qb) for q, qb in enumerate(queries)]
    got = run(batch)
    _same(got, run(seq), "batch")
    _same(got, run(orc), "batch")
    assert all(len(c) > 0 for c, _, _ in got)
    batch.close(); seq.close(); V.close()


def test_add_device_with_compaction(gpu_required):
    """Batches of two keyframes into a database held near max_postings, with erases leaving holes: the batch compacts the
    store when its rows do not fit behind the tail, and results equal host adds and the oracle at every step."""
    V = B.Vocabulary(flat_vocabulary(3000))
    rng = np.random.default_rng(8)
    P, K = 1000, 8

    def bow(n):
        ids = np.sort(rng.choice(3000, n, replace=False)).astype(np.int32)
        v = rng.uniform(0.1, 1, n)
        return ids, v / v.sum()

    dev_db, host_db, orc = B.KeyFrameDatabase(V, K, P), B.KeyFrameDatabase(V, K, P), OracleDB(K)
    first = [bow(n) for n in (250, 250, 200, 150, 150)]
    RowTable(first).add(dev_db, np.arange(5), np.arange(5))
    for s, b in enumerate(first):
        host_db.add(s, *b)
        orc.add(s, *b)
    assert dev_db.size() == host_db.size() == (5, P)
    occupied = list(range(5))
    for cyc in range(30):
        # erase two keyframes, and more until 200 postings are free
        n_erase = 0
        while n_erase < 2 or P - dev_db.size()[1] < 200:
            s = int(rng.choice(occupied))
            for o in (dev_db, host_db, orc):
                o.erase(s)
            occupied.remove(s)
            n_erase += 1
        free = P - dev_db.size()[1]
        n1 = int(rng.integers(20, free // 2))
        b1, b2 = bow(n1), bow(int(rng.integers(20, free - n1 + 1)))
        new = [int(x) for x in rng.choice([s for s in range(K) if s not in occupied], 2, replace=False)]
        RowTable([b1, b2]).add(dev_db, new, [0, 1])
        for s, b in zip(new, (b1, b2)):
            host_db.add(s, *b)
            orc.add(s, *b)
        occupied += new
        assert dev_db.size() == host_db.size()
        qb = bow(200)
        got = [dev_db.detect(1, *qb), dev_db.detect(0, *qb, [], 0.0)]
        _same(got, [host_db.detect(1, *qb), host_db.detect(0, *qb, [], 0.0)], cyc)
        _same(got, [orc.detect(1, *qb), orc.detect(0, *qb, [], 0.0)], cyc)
    dev_db.close(); host_db.close(); V.close()


def test_add_device_errors_leave_the_database_unchanged(gpu_required):
    """Over capacity (a batch whose first row alone would fit), an occupied, repeated or out-of-range slot, and rows whose count
    or ids are malformed: the call fails and the database keeps its size and its query results."""
    V = B.Vocabulary(flat_vocabulary(3000))
    rng = np.random.default_rng(4)

    def bow(n):
        ids = np.sort(rng.choice(3000, n, replace=False)).astype(np.int32)
        return ids, rng.uniform(0.1, 1, n)

    K, P = 4, 100
    db, twin, orc = B.KeyFrameDatabase(V, K, P), B.KeyFrameDatabase(V, K, P), OracleDB(K)
    b0 = bow(30)
    RowTable([b0]).add(db, [0], [0])
    twin.add(0, *b0)
    orc.add(0, *b0)
    good = bow(20)
    unsorted = (good[0][::-1].copy(), good[1])
    repeated = (np.concatenate([good[0][:10], good[0][9:19]]), good[1])
    too_big = (np.concatenate([good[0][:19], [3000]]).astype(np.int32), good[1])
    negative = (np.concatenate([[-1], good[0][1:]]).astype(np.int32), good[1])
    rows = [good, bow(50), bow(25), unsorted, repeated, too_big, negative, good, good]
    table = RowTable(rows, cap=64, n_override=[20, 50, 25, 20, 20, 20, 20, 65, -1])
    cases = [([1, 2], [1, 2], fe.ORBFE_ERR_CAPACITY),    # 30 + 50 fit, + 25 do not
             ([0], [0], fe.ORBFE_ERR_ARG),               # occupied
             ([1, 1], [0, 0], fe.ORBFE_ERR_ARG),         # repeated slot
             ([1, 4], [0, 0], fe.ORBFE_ERR_ARG),         # out of range
             ([1, 2], [0, 3], fe.ORBFE_ERR_ARG),         # ids descending
             ([1, 2], [0, 4], fe.ORBFE_ERR_ARG),         # an id twice
             ([1, 2], [0, 5], fe.ORBFE_ERR_ARG),         # an id >= the word count
             ([1, 2], [0, 6], fe.ORBFE_ERR_ARG),         # a negative id
             ([1, 2], [0, 7], fe.ORBFE_ERR_ARG),         # count > cap
             ([1, 2], [0, 8], fe.ORBFE_ERR_ARG)]         # count < 0
    qi = np.unique(np.concatenate([b0[0][:20], good[0][:10]])).astype(np.int32)
    q = (qi, np.full(len(qi), 1.0 / len(qi)))
    for slots, frames, code in cases:
        with pytest.raises(fe.OrbfeError) as e:
            table.add(db, slots, frames)
        assert e.value.code == code, (slots, frames)
        assert db.size() == (1, 30), (slots, frames)
        got = [db.detect(1, *q)]
        _same(got, [twin.detect(1, *q)], (slots, frames))
        _same(got, [orc.detect(1, *q)], (slots, frames))
    # and the database still takes a valid batch
    table.add(db, [2, 1], [0, 2])
    for o in (twin, orc):
        o.add(2, *good)
        o.add(1, *rows[2])
    assert db.size() == twin.size() == (3, 75)
    got = [db.detect(1, *q), db.detect(0, *q, [2], 0.0)]
    _same(got, [twin.detect(1, *q), twin.detect(0, *q, [2], 0.0)], "after")
    _same(got, [orc.detect(1, *q), orc.detect(0, *q, [2], 0.0)], "after")
    db.close(); twin.close(); V.close()


# ---- the whole chain ----------------------------------------------------------------------------------------------------
def test_chain_extract_bow_vector_add_detect_search(gpu_required):
    """extract_batch_device -> descend_device -> bow_vector_device + feature_vector_device -> add_device (slot = frame-store
    index) -> detect_device on frame 0's padded row -> search_by_bow_device on the candidates: nothing is copied to the host
    before the candidate count.  Equal to the host path: orbfe_bow_transform on the downloaded descriptors, host adds and
    detection on a twin database, the oracle, and the host orbfe_search_by_bow."""
    import torch
    from orb_slam_b200 import matching as M
    from orb_slam_b200.synth import textured_frame, shifted_frame
    dev = torch.device("cuda", 0)
    W, H, NF, levelsup = 640, 480, 1000, 3
    base = textured_frame(W, H, seed=11)
    frames = np.stack([base] + [shifted_frame(base, 3 * i - 12, 2 - i, seed=i) for i in range(1, 9)] +
                      [textured_frame(W, H, seed=100 + i) for i in range(4)])
    Bn = len(frames)
    voc = random_vocabulary(10, 4, seed=6)
    V = B.Vocabulary(voc)
    ex = fe.ORBextractor(NF, 1.2, 8)
    m = fe.ORBmatcher(0.75, True)
    s = torch.cuda.Stream(device=dev)
    z = lambda *shape: torch.zeros(shape, dtype=torch.int32, device=dev)
    d_frames = torch.from_numpy(frames).to(dev)
    d_valid = torch.from_numpy((np.random.default_rng(2).random((Bn, NF)) < 0.9).astype(np.uint8)).to(dev)
    d_kps = torch.zeros((Bn, NF, 28), dtype=torch.uint8, device=dev)
    d_desc = torch.zeros((Bn, NF, 32), dtype=torch.uint8, device=dev)
    d_cnt, d_leaf, d_node = z(Bn), z(Bn * NF), z(Bn * NF)
    d_ids, d_ptr, d_items, d_n = z(Bn, NF), z(Bn, NF + 1), z(Bn, NF), z(Bn)
    d_bids, d_bn = z(Bn, NF), z(Bn)
    d_bvals = torch.zeros((Bn, NF), dtype=torch.float64, device=dev)
    d_cand, d_nc, d_words = z(Bn), z(1), z(Bn)
    d_score = torch.zeros(Bn, dtype=torch.float32, device=dev)
    db, twin, orc = B.KeyFrameDatabase(V, Bn, Bn * NF), B.KeyFrameDatabase(V, Bn, Bn * NF), OracleDB(Bn)
    lists = {f: [g for g in (f - 1, f + 1) if 1 <= g < Bn] for f in range(1, Bn)}
    torch.cuda.synchronize()
    ss = s.cuda_stream
    ex.extract_batch_device(d_frames.data_ptr(), W, H, W, W * H, Bn, d_kps.data_ptr(), d_desc.data_ptr(), d_cnt.data_ptr(), ss)
    V.descend_device(d_desc.data_ptr(), Bn * NF, levelsup, d_leaf.data_ptr(), d_node.data_ptr(), ss)
    B.bow_vector_device(V, Bn, d_leaf.data_ptr(), d_cnt.data_ptr(), NF, d_bids.data_ptr(), d_bvals.data_ptr(), d_bn.data_ptr(), ss)
    B.feature_vector_device(V, Bn, d_leaf.data_ptr(), d_node.data_ptr(), d_cnt.data_ptr(), NF, d_ids.data_ptr(), d_ptr.data_ptr(),
                            d_items.data_ptr(), d_n.data_ptr(), ss)
    db.add_device(np.arange(1, Bn), np.arange(1, Bn), NF, d_bids.data_ptr(), d_bvals.data_ptr(), d_bn.data_ptr(), ss)
    db.set_covisibles(lists)
    db.detect_device(1, NF, d_bids.data_ptr(), d_bvals.data_ptr(), 0, 0, 0.0, Bn, d_cand.data_ptr(), d_nc.data_ptr(), d_words.data_ptr(),
                     d_score.data_ptr(), ss)
    s.synchronize()
    nc = int(d_nc.item())
    assert nc > 0
    d_i2 = z(nc)   # frame 0, the current frame
    d_out, d_nm = z(nc, NF), z(nc)
    M.search_by_bow_device(m, 0, nc, d_kps.data_ptr(), d_desc.data_ptr(), d_cnt.data_ptr(), NF, d_ids.data_ptr(), d_ptr.data_ptr(),
                           d_items.data_ptr(), d_n.data_ptr(), d_valid.data_ptr(), d_cand.data_ptr(), d_i2.data_ptr(), d_out.data_ptr(),
                           d_nm.data_ptr(), ss)
    s.synchronize()
    m.sync()
    cand = d_cand[:nc].cpu().numpy()
    # the host path
    desc, counts = d_desc.cpu().numpy(), d_cnt.cpu().numpy()
    bows = [V.transform(desc[f, :counts[f]], levelsup)[0] for f in range(Bn)]
    bids, bvals, bn = d_bids.cpu().numpy(), d_bvals.cpu().numpy(), d_bn.cpu().numpy()
    for f in range(Bn):
        check_row(bids[f], bvals[f], bn[f], *bows[f], ("chain", f))
    for o in (twin, orc):
        for f in range(1, Bn):
            o.add(f, *bows[f])
        o.set_covisibles(lists)
    hc, hw, hs = twin.detect(1, *bows[0])
    oc, _, _ = orc.detect(1, *bows[0])
    assert np.array_equal(cand, hc) and np.array_equal(cand, oc)
    assert np.array_equal(d_words.cpu().numpy(), hw) and np.array_equal(d_score.cpu().numpy().view(np.int32), hs.view(np.int32))
    assert any(1 <= c <= 8 for c in cand.tolist()), cand   # a keyframe of the current place
    kps = d_kps.cpu().numpy().view(fe.KP_DTYPE).reshape(Bn, NF)
    valid = d_valid.cpu().numpy()
    ids, ptr, items, n = (a.cpu().numpy() for a in (d_ids, d_ptr, d_items, d_n))
    fv = lambda f: (ids[f, :n[f]], ptr[f, :n[f] + 1], items[f, :ptr[f, n[f]]])
    out, nm = d_out.cpu().numpy(), d_nm.cpu().numpy()
    total = 0
    for j, f1 in enumerate(cand):
        n1, n2 = counts[f1], counts[0]
        n_h, out_h = M.search_by_bow(m, 0, desc[f1, :n1], valid[f1, :n1], kps[f1, :n1]["angle"], fv(f1), desc[0, :n2], valid[0, :n2],
                                     kps[0, :n2]["angle"], fv(0))
        assert nm[j] == n_h and np.array_equal(out[j, :n2], out_h), j
        total += n_h
    assert total > 50
    for o in (db, twin):
        o.close()
    ex.close(); V.close(); m.close()
