"""GPU tests of the device-resident keyframe database (include/orbfe_bow.h orbfe_kfdb_*): candidate lists (order included) and the
per-keyframe query fields equal the stateful oracle (oracle/kfdb.py) over whole sequences of add / erase / covisibility
refresh / clear / loop and relocalisation queries; the first query of a fresh database equals the stateless
orbfe_bow_db_detect; the device form equals the host form; capacity is exact and freed space is reused."""
import numpy as np
import pytest

import orb_slam_b200 as fe
from orb_slam_b200 import bow as B
from oracle.kfdb import KeyFrameDatabase as OracleDB

import kfdb_scenarios as S

pytestmark = pytest.mark.gpu


def flat_vocabulary(nwords):
    """A root with nwords leaf children: a vocabulary that only has to own the word ids 0 .. nwords-1."""
    n = nwords + 1
    child_ptr = np.zeros(n + 1, np.int32)
    child_ptr[1:] = nwords
    word_id = np.arange(-1, nwords, dtype=np.int32)
    return {"node_desc": np.zeros((n, 32), np.uint8), "child_ptr": child_ptr, "children": np.arange(1, n, dtype=np.int32),
            "word_id": word_id, "weight": np.ones(n), "L": 1}


def _same(got, want, tag):
    for q, ((gc, gw, gs), (wc, ww, ws)) in enumerate(zip(got, want)):
        assert np.array_equal(gc, wc), (tag, q, gc, wc)
        assert np.array_equal(gw, ww), (tag, q)
        assert np.array_equal(gs.view(np.int32), ws.view(np.int32)), (tag, q)   # bit for bit
    assert len(got) == len(want)


@pytest.fixture(scope="module")
def voc():
    V = B.Vocabulary(flat_vocabulary(3000))
    yield V
    V.close()


@pytest.mark.parametrize("seed", [0, 1, 2, 3])
def test_mixed_sequences_equal_the_oracle(gpu_required, voc, seed):
    ops, K = S.mixed_sequence(seed)
    db = B.KeyFrameDatabase(voc, K, 1 << 16)
    _same(S.replay(db, ops), S.replay(OracleDB(K), ops), seed)
    db.close()


def test_stale_reloc_score_is_read(gpu_required, voc):
    """The second relocalisation query accumulates the score the first one left in keyframe B (below the word threshold
    this time): the candidate is B, where the stateless orbfe_bow_db_detect (which counts such a score as 0) returns A."""
    ops = S.stale_reloc_sequence()
    db = B.KeyFrameDatabase(voc, 3, 1000)
    got = S.replay(db, ops)
    _same(got, S.replay(OracleDB(3), ops), "stale")
    assert list(got[1][0]) == [1]
    m = fe.ORBmatcher(0.75, True)
    adds = [op for op in ops if op[0] == "add"]
    kf_ptr = np.cumsum([0] + [len(op[2]) for op in adds]).astype(np.int32)
    covis = {0: [1], 1: [0], 2: []}
    cp = np.cumsum([0] + [len(covis[k]) for k in range(3)]).astype(np.int32)
    cand, _, _ = B.db_detect(m, 1, ops[-1][1], ops[-1][2], kf_ptr, np.concatenate([op[2] for op in adds]),
                             np.concatenate([op[3] for op in adds]), np.zeros(3, np.uint8), cp, np.array([1, 0], np.int32))
    assert list(cand) == [0]
    m.close()
    db.close()


@pytest.mark.parametrize("seed", [0, 1])
def test_first_query_equals_stateless_detect(gpu_required, seed):
    from orb_slam_b200.synth import random_keyframe_db
    d = random_keyframe_db(nkf=150, nwords=4000, words_per_kf=250, seed=seed, loop_at=30)
    V = B.Vocabulary(flat_vocabulary(4000))
    m = fe.ORBmatcher(0.75, True)
    nkf = len(d["kf_ptr"]) - 1
    lists = {k: list(d["covis"][d["covis_ptr"][k]:d["covis_ptr"][k + 1]]) for k in range(nkf)}
    for mode, min_score in ((0, 0.0), (0, 0.02), (1, 0.0)):
        db = B.KeyFrameDatabase(V, nkf, nkf * 250)
        for k in range(nkf):
            a, b = d["kf_ptr"][k], d["kf_ptr"][k + 1]
            db.add(k, d["db_ids"][a:b], d["db_vals"][a:b])
        db.set_covisibles(lists)
        conn = np.flatnonzero(d["connected"]) if mode == 0 else []
        cand, words, score = db.detect(mode, d["q_ids"], d["q_vals"], conn, min_score)
        c2, common, s2 = B.db_detect(m, mode, d["q_ids"], d["q_vals"], d["kf_ptr"], d["db_ids"], d["db_vals"], d["connected"],
                                     d["covis_ptr"], d["covis"], min_score)
        assert np.array_equal(cand, c2) and len(cand) > 0, (mode, min_score)
        assert np.array_equal(np.where(words < 0, 0, words), common)
        scored = s2 != -1
        assert scored.any() and np.array_equal(score[scored].view(np.int32), s2[scored].view(np.int32))
        db.close()
    m.close()
    V.close()


def test_device_form_equals_host_form(gpu_required, voc):
    import torch
    dev = torch.device("cuda", 0)
    ops, K = S.mixed_sequence(5)
    host, devdb = B.KeyFrameDatabase(voc, K, 1 << 16), B.KeyFrameDatabase(voc, K, 1 << 16)
    want = S.replay(host, ops)
    stream = torch.cuda.Stream(device=dev)
    got = []
    d_cand, d_n = torch.zeros(K, dtype=torch.int32, device=dev), torch.zeros(1, dtype=torch.int32, device=dev)
    d_words, d_score = torch.zeros(K, dtype=torch.int32, device=dev), torch.zeros(K, dtype=torch.float32, device=dev)
    for op in ops:
        if op[0] in ("loop", "reloc"):
            mode = 0 if op[0] == "loop" else 1
            qi = torch.from_numpy(np.ascontiguousarray(op[1], np.int32)).to(dev)
            qv = torch.from_numpy(np.ascontiguousarray(op[2], np.float64)).to(dev)
            conn = np.ascontiguousarray(op[3] if mode == 0 else [], np.int32)
            dc = torch.from_numpy(conn if len(conn) else np.zeros(1, np.int32)).to(dev)
            torch.cuda.synchronize()
            devdb.detect_device(mode, len(op[1]), qi.data_ptr(), qv.data_ptr(), len(conn), dc.data_ptr(), op[4] if mode == 0 else 0.0, K,
                                d_cand.data_ptr(), d_n.data_ptr(), d_words.data_ptr(), d_score.data_ptr(), stream.cuda_stream)
            stream.synchronize()
            n = int(d_n.item())
            got.append((d_cand[:n].cpu().numpy(), d_words.cpu().numpy(), d_score.cpu().numpy()))
        else:
            S.replay(devdb, [op])
    _same(got, want, "device")
    host.close()
    devdb.close()


def test_capacity_is_exact_and_space_is_reused(gpu_required, voc):
    rng = np.random.default_rng(3)
    P, K = 1000, 16
    db, orc = B.KeyFrameDatabase(voc, K, P), OracleDB(K)

    def bow(n):
        ids = np.sort(rng.choice(3000, n, replace=False)).astype(np.int32)
        v = rng.uniform(0.1, 1, n)
        return ids, v / v.sum()

    sizes = [300, 300, 250, 150]               # exactly P postings
    bows = [bow(n) for n in sizes]
    for s, (i, v) in enumerate(bows):
        db.add(s, i, v)
        orc.add(s, i, v)
    assert db.size() == (4, P)
    extra = bow(1)
    with pytest.raises(fe.OrbfeError) as e:
        db.add(5, *extra)
    assert e.value.code == fe.ORBFE_ERR_CAPACITY and db.size() == (4, P)
    q = (bows[1][0], bows[1][1])
    _same([db.detect(1, *q)], [orc.detect(1, *q)], "full")
    # add / erase cycles whose total is many times P: erased space is reused (holes are compacted)
    for cyc in range(60):
        s = int(rng.integers(0, 4))
        db.erase(s)
        orc.erase(s)
        n = int(rng.integers(100, 200 + sizes[s]))
        n = min(n, P - db.size()[1])
        b = bow(n)
        db.add(s, *b)
        orc.add(s, *b)
        qb = bow(200)
        _same([db.detect(1, *qb), db.detect(0, *qb, [], 0.0)], [orc.detect(1, *qb), orc.detect(0, *qb, [], 0.0)], cyc)
    db.close()


def test_handle_checks_leave_the_database_unchanged(gpu_required, voc):
    db = B.KeyFrameDatabase(voc, 4, 100)
    ids, vals = np.array([1, 5, 9], np.int32), np.array([0.2, 0.3, 0.5])
    db.add(0, ids, vals)
    for slot, i in ((4, ids), (0, ids), (1, np.array([1, 5, 3000], np.int32))):   # out of range, occupied, word id >= words
        with pytest.raises(fe.OrbfeError) as e:
            db.add(slot, i, vals)
        assert e.value.code == fe.ORBFE_ERR_ARG
    with pytest.raises(fe.OrbfeError):
        db.set_covisibles({0: [4]})
    with pytest.raises(fe.OrbfeError):
        db.detect(0, ids, vals, [7])
    with pytest.raises(fe.OrbfeError):
        db.detect(1, np.array([3000], np.int32), np.array([1.0]))
    assert db.size() == (1, 3)
    db.erase(3)                                 # empty slot: nothing to do
    cand, words, score = db.detect(1, ids, vals)
    assert list(cand) == [0] and words[0] == 3 and score[0] == np.float32(1.0)
    with pytest.raises(fe.OrbfeError) as e:     # more candidates than cap
        db.detect(1, ids, vals, cap=0)
    assert e.value.code == fe.ORBFE_ERR_CAPACITY
    db.close()


def test_large_seeded_database(gpu_required):
    """10k keyframes of 200 words each, word ids spread over 10^6 (the size of the ORB vocabulary), loop and relocalisation
    queries interleaved with erases and re-adds."""
    rng = np.random.default_rng(11)
    NW, NKF, WPK = 1_000_000, 10_000, 200
    V = B.Vocabulary(flat_vocabulary(NW))
    bows, at = S.trajectory(NKF + 500, NW, WPK, seed=4, shift=20)
    db, orc = B.KeyFrameDatabase(V, NKF, NKF * WPK), OracleDB(NKF)
    lists = {}
    for k in range(NKF):
        db.add(k, *bows[k])
        orc.add(k, *bows[k])
        lists[k] = [j for j in (k - 1, k + 1, k - 2, k + 2, k - 3, k + 3) if 0 <= j < NKF][:int(rng.integers(0, 7))]
    db.set_covisibles(lists)
    orc.set_covisibles(lists)
    got, want = [], []
    for it in range(30):
        src = int(rng.integers(0, NKF))
        q = at(20 * src + int(rng.integers(0, 10)), 555 + it)
        conn = [j for j in range(src - 3, src + 4) if 0 <= j < NKF and j != src]
        got.append(db.detect(it % 2, *q, conn, 0.0))
        want.append(orc.detect(it % 2, *q, conn, 0.0))
        if it % 5 == 4:   # erase a keyframe (its neighbours forget it) and put a new one in its slot
            s = int(rng.integers(0, NKF))
            for o in (db, orc):
                o.erase(s)
            fix = {o: [x for x in lists[o] if x != s] for o in lists if s in lists[o]}
            lists.update(fix)
            b = bows[NKF + it]
            for o in (db, orc):
                o.set_covisibles(fix) if fix else None
                o.add(s, *b)
    _same(got, want, "large")
    assert all(len(c) > 0 for c, _, _ in got)
    db.close()
    V.close()


def test_chain_extract_transform_add_detect_search(gpu_required):
    """Extraction -> orbfe_bow_transform -> add of the keyframes (slot = frame-store index) -> device relocalisation detection ->
    orbfe_search_by_bow_device on the returned slots, the candidates never leaving the device; equal to the host path (the
    host-form detection on a twin database, the oracle, and the host orbfe_search_by_bow on the downloaded arrays)."""
    import torch
    from orb_slam_b200 import matching as M
    from orb_slam_b200.synth import textured_frame, shifted_frame, random_vocabulary
    dev = torch.device("cuda", 0)
    W, H, NF, levelsup = 640, 480, 1000, 3
    base = textured_frame(W, H, seed=11)
    # frame 0: the current frame; 1..8 keyframes of the same place; 9..12 keyframes of other places
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
    torch.cuda.synchronize()
    ex.extract_batch_device(d_frames.data_ptr(), W, H, W, W * H, Bn, d_kps.data_ptr(), d_desc.data_ptr(), d_cnt.data_ptr(), s.cuda_stream)
    V.descend_device(d_desc.data_ptr(), Bn * NF, levelsup, d_leaf.data_ptr(), d_node.data_ptr(), s.cuda_stream)
    B.feature_vector_device(V, Bn, d_leaf.data_ptr(), d_node.data_ptr(), d_cnt.data_ptr(), NF, d_ids.data_ptr(), d_ptr.data_ptr(),
                            d_items.data_ptr(), d_n.data_ptr(), s.cuda_stream)
    s.synchronize()
    desc, counts = d_desc.cpu().numpy(), d_cnt.cpu().numpy()
    bows = [V.transform(desc[f, :counts[f]], levelsup)[0] for f in range(Bn)]
    db, twin, orc = B.KeyFrameDatabase(V, Bn, Bn * NF), B.KeyFrameDatabase(V, Bn, Bn * NF), OracleDB(Bn)
    lists = {f: [g for g in (f - 1, f + 1) if 1 <= g < Bn] for f in range(1, Bn)}
    for o in (db, twin, orc):
        for f in range(1, Bn):
            o.add(f, *bows[f])
        o.set_covisibles(lists)
    # device relocalisation detection, then SearchByBoW(KeyFrame*, Frame&) of every candidate against frame 0
    t = lambda a, dt: torch.from_numpy(np.ascontiguousarray(a, dt)).to(dev)
    d_qi, d_qv = t(bows[0][0], np.int32), t(bows[0][1], np.float64)
    d_cand, d_nc = z(Bn), z(1)
    db.detect_device(1, len(bows[0][0]), d_qi.data_ptr(), d_qv.data_ptr(), 0, 0, 0.0, Bn, d_cand.data_ptr(), d_nc.data_ptr(),
                     stream=s.cuda_stream)
    s.synchronize()
    nc = int(d_nc.item())
    assert nc > 0
    d_i2 = z(nc)   # frame 0, the current frame
    d_out, d_nm = z(nc, NF), z(nc)
    M.search_by_bow_device(m, 0, nc, d_kps.data_ptr(), d_desc.data_ptr(), d_cnt.data_ptr(), NF, d_ids.data_ptr(), d_ptr.data_ptr(),
                           d_items.data_ptr(), d_n.data_ptr(), d_valid.data_ptr(), d_cand.data_ptr(), d_i2.data_ptr(), d_out.data_ptr(),
                           d_nm.data_ptr(), s.cuda_stream)
    s.synchronize()
    m.sync()
    cand = d_cand[:nc].cpu().numpy()
    # the host path
    hc, _, _ = twin.detect(1, *bows[0])
    oc, _, _ = orc.detect(1, *bows[0])
    assert np.array_equal(cand, hc) and np.array_equal(cand, oc)
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
