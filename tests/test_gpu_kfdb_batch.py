"""GPU tests of the batched keyframe-database query (include/orbfe_bow.h orbfe_kfdb_detect_batch_device): every scene of
kfdb_domain_scenes.py, kfdb_scenarios.py and kfdb_batch_scenes.py replayed with its runs of same-mode queries cut into batches
equals, bit for bit, a twin database answering one orbfe_kfdb_detect_device call at a time and the sequential oracle
(oracle/kfdb.py), including a single query after every batch (the state the batch left); the batch and cap limits; the
stream-ordering promise without host synchronisation; and extraction -> BowVectors -> one batched query -> one SearchByBoW
launch over every (candidate, frame) job equal to the same chain one frame at a time."""
import numpy as np
import pytest

import orb_slam_b200 as fe
from orb_slam_b200 import bow as B
from oracle.kfdb import KeyFrameDatabase as OracleDB

import kfdb_batch_scenes as BS
import kfdb_domain_scenes as S
import kfdb_scenarios as KS
from test_gpu_kfdb import flat_vocabulary, _same
from test_oracle_kfdb_batch import ALL

pytestmark = pytest.mark.gpu

SPIN = 100_000_000          # torch.cuda._sleep cycles: one bounded spin of roughly 50 ms on an H100
PAD = np.iinfo(np.int32).max


@pytest.fixture(scope="module")
def voc():
    V = B.Vocabulary(flat_vocabulary(S.NWORDS))
    yield V
    V.close()


def _torch():
    import torch
    return torch, torch.device("cuda", 0)


def _dev(a, dt):
    torch, dev = _torch()
    return torch.from_numpy(np.ascontiguousarray(a, dt)).to(dev)


def _rows(qops, qcap=None):
    """The queries as padded rows (ids PAD, values 0 past the real words), qcap = the longest row unless given."""
    qcap = max([len(op[1]) for op in qops]) if qcap is None else qcap
    ids, vals = np.full((len(qops), max(qcap, 1)), PAD, np.int32), np.zeros((len(qops), max(qcap, 1)))
    for b, op in enumerate(qops):
        ids[b, :len(op[1])], vals[b, :len(op[1])] = op[1], op[2]
    return qcap, ids, vals


class Enqueued:
    """One batch enqueued on a stream with its own inputs and outputs; result() after the stream is synchronised."""

    def __init__(self, db, qops, stream, fields=True, qcap=None, cap=None):
        torch, dev = _torch()
        K = db.max_keyframes
        self.n, self.K, self.cap = len(qops), K, K if cap is None else cap
        mode = 0 if qops[0][0] == "loop" else 1
        qcap, ids, vals = _rows(qops, qcap)
        self.keep = [_dev(ids, np.int32), _dev(vals, np.float64)]
        ptr, conn, ms = 0, 0, 0
        if mode == 0:
            flat = [c for op in qops for c in op[3]]
            self.keep += [_dev(np.cumsum([0] + [len(op[3]) for op in qops]), np.int32), _dev(np.array([op[4] for op in qops]), np.float32)]
            ptr, ms = self.keep[2].data_ptr(), self.keep[3].data_ptr()
            if flat:
                self.keep.append(_dev(flat, np.int32))
                conn = self.keep[-1].data_ptr()
        z = lambda n, dt: torch.zeros(max(n, 1), dtype=dt, device=dev)
        self.cand, self.ncand = z(self.n * self.cap, torch.int32), z(self.n, torch.int32)
        self.words = z(self.n * K, torch.int32) if fields else None
        self.score = z(self.n * K, torch.float32) if fields else None
        torch.cuda.current_stream().synchronize()
        db.detect_batch_device(mode, self.n, qcap, self.keep[0].data_ptr(), self.keep[1].data_ptr(), ptr, conn, ms, self.cap,
                               self.cand.data_ptr(), self.ncand.data_ptr(), self.words.data_ptr() if fields else 0,
                               self.score.data_ptr() if fields else 0, stream.cuda_stream)

    def result(self):
        cand, nc = self.cand.cpu().numpy(), self.ncand.cpu().numpy()
        K = self.K
        w = self.words.cpu().numpy() if self.words is not None else np.full(self.n * K, -1, np.int32)
        s = self.score.cpu().numpy() if self.score is not None else np.full(self.n * K, -1, np.float32)
        return [(cand[b * self.cap:b * self.cap + min(nc[b], self.cap)], w[b * K:(b + 1) * K], s[b * K:(b + 1) * K]) for b in range(self.n)]


class DeviceDB:
    """The library database driven through detect_batch_device (batched) or one detect_device call per query (single)."""

    def __init__(self, voc, K, P, max_queries, single=False, fields=True):
        torch, dev = _torch()
        self.db = B.KeyFrameDatabase(voc, K, P, max_queries)
        self.single, self.fields, self.K = single, fields, K
        self.stream = torch.cuda.Stream(device=dev)

    def __getattr__(self, name):            # add / erase / clear / set_covisibles
        return getattr(self.db, name)

    def detect_batch(self, mode, qops):
        if self.single:
            return [self.detect_one(op) for op in qops]
        e = Enqueued(self.db, qops, self.stream, self.fields)
        self.stream.synchronize()
        return e.result()

    def detect_one(self, op):
        torch, dev = _torch()
        mode = 0 if op[0] == "loop" else 1
        K = self.K
        qi, qv = _dev(op[1] if len(op[1]) else [0], np.int32), _dev(op[2] if len(op[2]) else [0.0], np.float64)
        conn = op[3] if mode == 0 else []
        dc = _dev(conn, np.int32) if len(conn) else None
        d_cand, d_n = torch.zeros(K, dtype=torch.int32, device=dev), torch.zeros(1, dtype=torch.int32, device=dev)
        d_w, d_s = torch.zeros(K, dtype=torch.int32, device=dev), torch.zeros(K, dtype=torch.float32, device=dev)
        torch.cuda.current_stream().synchronize()
        self.db.detect_device(mode, len(op[1]), qi.data_ptr(), qv.data_ptr(), len(conn), dc.data_ptr() if dc is not None else 0,
                              op[4] if mode == 0 else 0.0, K, d_cand.data_ptr(), d_n.data_ptr(), d_w.data_ptr(), d_s.data_ptr(),
                              self.stream.cuda_stream)
        self.stream.synchronize()
        return d_cand[:int(d_n.item())].cpu().numpy(), d_w.cpu().numpy(), d_s.cpu().numpy()

    def detect(self, mode, q_ids, q_vals, connected=(), min_score=0.0):
        return self.detect_one(("loop", q_ids, q_vals, list(connected), min_score) if mode == 0 else ("reloc", q_ids, q_vals))


class SequentialOracle(OracleDB):
    def detect_batch(self, mode, qops):
        return KS.replay(self, qops)


def _with_probes(db, ops, size):
    """replay_batched, and after every batch one single query (a copy of the batch's last query) whose result depends on the
    persistent scores the batch left."""
    out = []
    for kind, item in BS.runs(ops):
        if kind == "op":
            KS.replay(db, [item])
            continue
        n = size or len(item)
        for i in range(0, len(item), n):
            chunk = item[i:i + n]
            out += db.detect_batch(0 if chunk[0][0] == "loop" else 1, chunk)
            out += KS.replay(db, [chunk[-1]]) if not isinstance(db, DeviceDB) else [db.detect_one(chunk[-1])]
    return out


def _P(ops):
    live, peak = {}, 1
    for op in ops:
        if op[0] == "add":
            live[op[1]] = len(op[2])
        elif op[0] == "erase":
            live.pop(op[1], None)
        elif op[0] == "clear":
            live.clear()
        peak = max(peak, sum(live.values()))
    return peak


@pytest.mark.parametrize("name,ops,K", ALL, ids=[a[0] for a in ALL])
def test_scene_batches_equal_single_calls_and_the_oracle(gpu_required, voc, name, ops, K):
    longest = max(BS.longest_run(ops), 1)
    P = _P(ops)
    twin = DeviceDB(voc, K, P, 1, single=True)
    try:
        single = _with_probes(twin, ops, 1)
    finally:
        twin.close()
    sizes = [(1, 1), (2, 2), (None, longest)] + ([(3, 3)] if longest > 3 else [])
    for size, mq in sizes:
        want = _with_probes(SequentialOracle(K), ops, size)
        db = DeviceDB(voc, K, P, mq)
        try:
            got = _with_probes(db, ops, size)
        finally:
            db.close()
        _same(got, want, "%s size %s" % (name, size))
        if size == 1:
            _same(single, want, name + " single calls")
    bare = DeviceDB(voc, K, P, longest, fields=False)         # d_words / d_score NULL: the same candidates
    try:
        got = BS.replay_batched(bare, ops, None)
    finally:
        bare.close()
    want = KS.replay(OracleDB(K), ops)
    assert len(got) == len(want)
    for q, ((gc, _, _), (wc, _, _)) in enumerate(zip(got, want)):
        assert np.array_equal(gc, wc), (name, q)


# ---- limits ------------------------------------------------------------------------------------------------------------------------
def test_max_queries_accepted_and_one_more_refused(gpu_required, voc):
    """B = max_queries runs; B = max_queries + 1 is ORBFE_ERR_ARG before any work, and the database answers on as if it had
    not been called."""
    torch, dev = _torch()
    sc = BS.shared_candidate(16)
    qops = [op for op in sc.ops if op[0] == "reloc"]
    want = KS.replay(OracleDB(sc.K), sc.ops)
    db = DeviceDB(voc, sc.K, sc.P, 8)
    try:
        KS.replay(db, [op for op in sc.ops if op[0] not in ("loop", "reloc")])
        with pytest.raises(fe.OrbfeError) as e:
            Enqueued(db.db, qops[:9], db.stream)
        assert e.value.code == fe.ORBFE_ERR_ARG
        got = db.detect_batch(1, qops[:8]) + db.detect_batch(1, qops[8:])
    finally:
        db.close()
    _same(got, want, "max_queries")
    for M in (1, 1024):
        B.KeyFrameDatabase(voc, 4, 16, M).close()


def test_per_query_cap(gpu_required, voc):
    """Three relocalisation rows of the 2049-keyframe scene (over a thousand candidates each) with cap 0, 1, n-1, n and n+1:
    every count is n, every row holds the first min(cap, n) candidates, and nothing is written past the last row."""
    torch, dev = _torch()
    sc = S.sizes(2049)
    op = next(op for op in sc.ops if op[0] == "reloc")
    want = KS.replay(OracleDB(sc.K), [o for o in sc.ops if o[0] == "add"] + [op])[0][0]
    n = len(want)
    assert n > 1024
    db = B.KeyFrameDatabase(voc, sc.K, sc.P, 3)
    st = torch.cuda.Stream(device=dev)
    GUARD = -7
    try:
        KS.replay(db, [o for o in sc.ops if o[0] == "add"])
        _, ids, vals = _rows([op] * 3)
        d_ids, d_vals = _dev(ids, np.int32), _dev(vals, np.float64)
        for cap in (0, 1, n - 1, n, n + 1):
            d_cand = torch.full((3 * cap + 16,), GUARD, dtype=torch.int32, device=dev)
            d_n = torch.full((3,), GUARD, dtype=torch.int32, device=dev)
            torch.cuda.synchronize()
            db.detect_batch_device(1, 3, ids.shape[1], d_ids.data_ptr(), d_vals.data_ptr(), 0, 0, 0, cap, d_cand.data_ptr(), d_n.data_ptr(),
                                   stream=st.cuda_stream)
            st.synchronize()
            got, nc = d_cand.cpu().numpy(), d_n.cpu().numpy()
            k = min(cap, n)
            assert nc.tolist() == [n] * 3, cap
            for b in range(3):
                assert np.array_equal(got[b * cap:b * cap + k], want[:k]), (cap, b)
            assert np.all(got[3 * cap:] == GUARD), cap
    finally:
        db.close()


def test_qcap_65535_padded_rows(gpu_required, voc):
    """The two_scorers batch passed as rows of 65535 entries, nearly all padding: the oracle's results."""
    torch, dev = _torch()
    sc = BS.two_scorers()
    qops = [op for op in sc.ops if op[0] == "reloc"]
    want = KS.replay(OracleDB(sc.K), sc.ops)
    db = DeviceDB(voc, sc.K, sc.P, 3)
    try:
        KS.replay(db, [op for op in sc.ops if op[0] not in ("loop", "reloc")])
        e = Enqueued(db.db, qops, db.stream, qcap=65535)
        db.stream.synchronize()
        got = e.result()
    finally:
        db.close()
    _same(got, want, "qcap 65535")


def test_64_relocalisations_against_10000_keyframes(gpu_required, voc):
    """64 relocalisation queries in one batch on a database of 10,000 trajectory keyframes equal 64 detect_device calls on a
    twin database (candidates, words, scores), and most queries have candidates."""
    bows, at = KS.trajectory(10000, S.NWORDS, 150, seed=4)
    K = len(bows)
    lists = {k: [j for j in (k - 1, k + 1, k - 2, k + 2, k - 3, k + 3) if 0 <= j < K] for k in range(K)}
    rng = np.random.default_rng(9)
    qops = [("reloc", *at(int(rng.integers(0, K)) * max(1, 150 // 8) + 3, 500 + i)) for i in range(64)]
    P = sum(len(b[0]) for b in bows)
    dbs = [DeviceDB(voc, K, P, 64), DeviceDB(voc, K, P, 1, single=True)]
    try:
        for d in dbs:
            for k, bw in enumerate(bows):
                d.add(k, *bw)
            d.set_covisibles(lists)
        got, want = dbs[0].detect_batch(1, qops), dbs[1].detect_batch(1, qops)
        # the state each left: one more query that reads stale scores
        got.append(dbs[0].detect_one(qops[0]))
        want.append(dbs[1].detect_one(qops[0]))
    finally:
        for d in dbs:
            d.close()
    _same(got, want, "10k")
    assert sum(len(c) > 0 for c, _, _ in got) >= 32


# ---- stream ordering -------------------------------------------------------------------------------------------------------------
def test_batch_behind_add_device_and_query_rows_behind_spins(gpu_required, voc):
    """Keyframe rows copied on stream A behind a spin and added with add_device(stream A); then the query rows copied on stream
    C behind another spin and the batch enqueued on C at once; one synchronisation at the end."""
    torch, dev = _torch()
    sc = S.sizes(1025)
    adds = [op for op in sc.ops if op[0] == "add"]
    qops = [op for op in sc.ops if op[0] == "reloc"] * 3
    cap = max(len(a[2]) for a in adds)
    ids, vals = np.full((len(adds), cap), PAD, np.int32), np.zeros((len(adds), cap))
    for r, a in enumerate(adds):
        ids[r, :len(a[2])], vals[r, :len(a[2])] = a[2], a[3]
    counts = np.array([len(a[2]) for a in adds], np.int32)
    src = (_dev(ids, np.int32), _dev(vals, np.float64), _dev(counts, np.int32))
    dst = tuple(torch.zeros_like(t) for t in src)
    qcap, qi, qv = _rows(qops)
    qsrc, qdst = (_dev(qi, np.int32), _dev(qv, np.float64)), (torch.zeros(qi.shape, dtype=torch.int32, device=dev),
                                                               torch.zeros(qv.shape, dtype=torch.float64, device=dev))
    want = KS.replay(OracleDB(sc.K), adds + qops)
    db = B.KeyFrameDatabase(voc, sc.K, sc.P, 3)
    try:
        A, Cs = torch.cuda.Stream(device=dev), torch.cuda.Stream(device=dev)
        d_cand, d_n = torch.zeros(3 * sc.K, dtype=torch.int32, device=dev), torch.zeros(3, dtype=torch.int32, device=dev)
        d_w, d_s = torch.zeros(3 * sc.K, dtype=torch.int32, device=dev), torch.zeros(3 * sc.K, dtype=torch.float32, device=dev)
        torch.cuda.synchronize()
        with torch.cuda.stream(A):
            torch.cuda._sleep(SPIN)
            for d, s in zip(dst, src):
                d.copy_(s)
        db.add_device([a[1] for a in adds], np.arange(len(adds)), cap, dst[0].data_ptr(), dst[1].data_ptr(), dst[2].data_ptr(),
                      stream=A.cuda_stream)
        with torch.cuda.stream(Cs):
            torch.cuda._sleep(SPIN)
            for d, s in zip(qdst, qsrc):
                d.copy_(s)
        db.detect_batch_device(1, 3, qcap, qdst[0].data_ptr(), qdst[1].data_ptr(), 0, 0, 0, sc.K, d_cand.data_ptr(), d_n.data_ptr(),
                               d_w.data_ptr(), d_s.data_ptr(), Cs.cuda_stream)
        torch.cuda.synchronize()
        c, n, w, s = (t.cpu().numpy() for t in (d_cand, d_n, d_w, d_s))
        K = sc.K
        got = [(c[b * K:b * K + n[b]], w[b * K:(b + 1) * K], s[b * K:(b + 1) * K]) for b in range(3)]
    finally:
        db.close()
    _same(got, want, "behind spins")


@pytest.mark.parametrize("kind", ["erase", "add", "covis", "clear"])
def test_host_call_waits_for_the_pending_batch(gpu_required, voc, kind):
    """A batch of two queries enqueued on stream A behind a spin, then at once a synchronous host call that would change the
    batch's results had it run first: the batch sees the database as it was; the next query sees the call."""
    torch, dev = _torch()
    sc = S.host_call(kind)
    op = sc.ops[sc.pending]
    ops = sc.ops[:sc.pending + 1] + [op] + sc.ops[sc.pending + 1:]
    want = KS.replay(OracleDB(sc.K), ops)
    db = DeviceDB(voc, sc.K, sc.P, 2)
    try:
        KS.replay(db, sc.ops[:sc.pending])
        A = torch.cuda.Stream(device=dev)
        torch.cuda.synchronize()
        with torch.cuda.stream(A):
            torch.cuda._sleep(SPIN)
        e = Enqueued(db.db, [op, op], A)
        KS.replay(db, [sc.ops[sc.pending + 1]])          # the host call, with the batch still pending
        A.synchronize()
        got = e.result() + KS.replay(db, sc.ops[sc.pending + 2:])
    finally:
        db.close()
    _same(got, want, kind)
    assert not np.array_equal(want[0][0], want[2][0])


def test_batch_chain_on_four_streams(gpu_required, voc):
    """The eight queries of stream_chain (each reads the score the one before left) as four batches of two, each on its own
    stream into its own buffers, behind a spin on the first stream; one synchronisation at the end."""
    torch, dev = _torch()
    sc = S.stream_chain(8)
    want = KS.replay(OracleDB(sc.K), sc.ops)
    qops = [op for op in sc.ops if op[0] == "reloc"]
    db = B.KeyFrameDatabase(voc, sc.K, sc.P, 2)
    try:
        KS.replay(db, [op for op in sc.ops if op[0] not in ("loop", "reloc")])
        streams = [torch.cuda.Stream(device=dev) for _ in range(4)]
        torch.cuda.synchronize()
        with torch.cuda.stream(streams[0]):
            torch.cuda._sleep(SPIN)
        pend = [Enqueued(db, qops[2 * i:2 * i + 2], streams[i]) for i in range(4)]
        torch.cuda.synchronize()
        got = sum((p.result() for p in pend), [])
    finally:
        db.close()
    _same(got, want, "chain")


# ---- end to end -------------------------------------------------------------------------------------------------------------------
def test_extract_bow_batch_detect_search_by_bow(gpu_required):
    """Four current frames and twelve keyframes extracted in one launch chain; BowVectors and FeatureVectors on the device; the
    keyframes added with add_device; the four frames' relocalisation queries as ONE detect_batch_device on the padded BowVector
    rows; ONE search_by_bow_device over every (candidate, frame) job.  The same chain one frame at a time (detect_device on a
    twin database, one search_by_bow_device per frame) gives the same candidates and the same matches."""
    torch, dev = _torch()
    from orb_slam_b200 import matching as M
    from orb_slam_b200.synth import random_vocabulary, shifted_frame, textured_frame
    W, H, NF, levelsup = 640, 480, 1000, 3
    bases = [textured_frame(W, H, seed=11), textured_frame(W, H, seed=12)]
    cur = [shifted_frame(bases[0], 2, 1, seed=40), shifted_frame(bases[1], -3, 2, seed=41), shifted_frame(bases[0], -1, -2, seed=42),
           textured_frame(W, H, seed=300)]
    kfs = [shifted_frame(bases[i % 2], 3 * i - 12, 2 - i, seed=i) for i in range(1, 9)] + [textured_frame(W, H, seed=100 + i) for i in range(4)]
    frames = np.stack(cur + kfs)
    NQ, Bn = len(cur), len(frames)
    V = B.Vocabulary(random_vocabulary(10, 4, seed=6))
    ex, m = fe.ORBextractor(NF, 1.2, 8), fe.ORBmatcher(0.75, True)
    s = torch.cuda.Stream(device=dev)
    z = lambda *shape: torch.zeros(shape, dtype=torch.int32, device=dev)
    d_frames = torch.from_numpy(frames).to(dev)
    d_valid = torch.from_numpy((np.random.default_rng(2).random((Bn, NF)) < 0.9).astype(np.uint8)).to(dev)
    d_kps, d_desc = torch.zeros((Bn, NF, 28), dtype=torch.uint8, device=dev), torch.zeros((Bn, NF, 32), dtype=torch.uint8, device=dev)
    d_cnt, d_leaf, d_node = z(Bn), z(Bn * NF), z(Bn * NF)
    d_ids, d_ptr, d_items, d_n = z(Bn, NF), z(Bn, NF + 1), z(Bn, NF), z(Bn)
    d_bid, d_bval, d_bn = z(Bn, NF), torch.zeros((Bn, NF), dtype=torch.float64, device=dev), z(Bn)
    torch.cuda.synchronize()
    ex.extract_batch_device(d_frames.data_ptr(), W, H, W, W * H, Bn, d_kps.data_ptr(), d_desc.data_ptr(), d_cnt.data_ptr(), s.cuda_stream)
    V.descend_device(d_desc.data_ptr(), Bn * NF, levelsup, d_leaf.data_ptr(), d_node.data_ptr(), s.cuda_stream)
    B.bow_vector_device(V, Bn, d_leaf.data_ptr(), d_cnt.data_ptr(), NF, d_bid.data_ptr(), d_bval.data_ptr(), d_bn.data_ptr(), s.cuda_stream)
    B.feature_vector_device(V, Bn, d_leaf.data_ptr(), d_node.data_ptr(), d_cnt.data_ptr(), NF, d_ids.data_ptr(), d_ptr.data_ptr(),
                            d_items.data_ptr(), d_n.data_ptr(), s.cuda_stream)
    slots = np.arange(NQ, Bn)
    lists = {f: [g for g in (f - 1, f + 1, f - 2, f + 2) if NQ <= g < Bn] for f in range(NQ, Bn)}
    db, twin = B.KeyFrameDatabase(V, Bn, Bn * NF, NQ), B.KeyFrameDatabase(V, Bn, Bn * NF)
    args = (NF, d_bid.data_ptr(), d_bval.data_ptr(), d_bn.data_ptr())
    try:
        for o in (db, twin):
            o.add_device(slots, slots, *args, stream=s.cuda_stream)
            o.set_covisibles(lists)
        # batched: one detection for the four frames, one SearchByBoW launch over every (candidate, frame) job
        d_cand, d_nc = z(NQ * Bn), z(NQ)
        db.detect_batch_device(1, NQ, NF, d_bid.data_ptr(), d_bval.data_ptr(), 0, 0, 0, Bn, d_cand.data_ptr(), d_nc.data_ptr(),
                               stream=s.cuda_stream)
        s.synchronize()
        nc = d_nc.cpu().numpy()
        cand = d_cand.cpu().numpy()
        jobs = [(int(c), f) for f in range(NQ) for c in cand[f * Bn:f * Bn + nc[f]]]
        assert len(jobs) >= NQ
        d_i1, d_i2 = _dev([j[0] for j in jobs], np.int32), _dev([j[1] for j in jobs], np.int32)
        d_out, d_nm = z(len(jobs), NF), z(len(jobs))
        M.search_by_bow_device(m, 0, len(jobs), d_kps.data_ptr(), d_desc.data_ptr(), d_cnt.data_ptr(), NF, d_ids.data_ptr(), d_ptr.data_ptr(),
                               d_items.data_ptr(), d_n.data_ptr(), d_valid.data_ptr(), d_i1.data_ptr(), d_i2.data_ptr(), d_out.data_ptr(),
                               d_nm.data_ptr(), s.cuda_stream)
        s.synchronize()
        m.sync()
        out, nm = d_out.cpu().numpy(), d_nm.cpu().numpy()
        # one frame at a time
        j = 0
        total = 0
        for f in range(NQ):
            c1, n1 = z(Bn), z(1)
            twin.detect_device(1, NF, d_bid[f].data_ptr(), d_bval[f].data_ptr(), 0, 0, 0.0, Bn, c1.data_ptr(), n1.data_ptr(),
                               stream=s.cuda_stream)
            s.synchronize()
            k = int(n1.item())
            assert k == nc[f] and np.array_equal(c1[:k].cpu().numpy(), cand[f * Bn:f * Bn + k]), f
            if k == 0:
                continue
            o1, m1 = z(k, NF), z(k)
            M.search_by_bow_device(m, 0, k, d_kps.data_ptr(), d_desc.data_ptr(), d_cnt.data_ptr(), NF, d_ids.data_ptr(), d_ptr.data_ptr(),
                                   d_items.data_ptr(), d_n.data_ptr(), d_valid.data_ptr(), c1.data_ptr(), _dev([f] * k, np.int32).data_ptr(),
                                   o1.data_ptr(), m1.data_ptr(), s.cuda_stream)
            s.synchronize()
            m.sync()
            assert np.array_equal(m1.cpu().numpy(), nm[j:j + k]) and np.array_equal(o1.cpu().numpy(), out[j:j + k]), f
            total += int(m1.sum().item())
            j += k
        assert j == len(jobs) and total > 50
    finally:
        db.close(); twin.close(); ex.close(); V.close(); m.close()
