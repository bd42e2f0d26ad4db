"""GPU tests of the resident keyframe database (include/orbfe_bow.h orbfe_kfdb_*) on the scenes of tests/kfdb_domain_scenes.py:
host form and device form equal the stateful oracle (oracle/kfdb.py) bit for bit on every scene, the device form's capacity
and nq limits, a database of 2^24 slots, and the promise that every call is ordered after the handle's previous work
whatever stream it was enqueued on (no host synchronisation between the calls of those tests)."""
import ctypes as C

import numpy as np
import pytest

import orb_slam_b200 as fe
from orb_slam_b200 import bow as B
from oracle.kfdb import KeyFrameDatabase as OracleDB

import kfdb_domain_scenes as S
import kfdb_scenarios as KS
from test_gpu_kfdb import flat_vocabulary, _same

pytestmark = pytest.mark.gpu

SPIN = 100_000_000          # torch.cuda._sleep cycles: one bounded spin of roughly 50 ms on an H100


@pytest.fixture(scope="module")
def voc():
    V = B.Vocabulary(flat_vocabulary(S.NWORDS))
    yield V
    V.close()


def _dev(a, dt):
    import torch
    return torch.from_numpy(np.ascontiguousarray(a, dt)).to(torch.device("cuda", 0))


def _zeros(n, dt):
    import torch
    return torch.zeros(max(n, 1), dtype=dt, device=torch.device("cuda", 0))


def _query_args(op):
    """(mode, device q_ids, device q_vals, nconn, device connected or None, min_score) of a query op, uploaded."""
    mode = 0 if op[0] == "loop" else 1
    conn = op[3] if mode == 0 else []
    return (mode, _dev(op[1], np.int32), _dev(op[2], np.float64), len(conn), _dev(conn, np.int32) if len(conn) else None,
            op[4] if mode == 0 else 0.0)


def _detect_device(db, K, op, stream, fields=True):
    import torch
    mode, qi, qv, nc, dc, ms = _query_args(op)
    d_cand, d_n = _zeros(K, torch.int32), _zeros(1, torch.int32)
    d_w, d_s = _zeros(K, torch.int32), _zeros(K, torch.float32)
    torch.cuda.synchronize()
    db.detect_device(mode, len(op[1]), qi.data_ptr(), qv.data_ptr(), nc, dc.data_ptr() if dc is not None else 0, ms, K, d_cand.data_ptr(),
                     d_n.data_ptr(), d_w.data_ptr() if fields else 0, d_s.data_ptr() if fields else 0, stream.cuda_stream)
    stream.synchronize()
    n = int(d_n.item())
    return d_cand[:n].cpu().numpy(), d_w[:K].cpu().numpy(), d_s[:K].cpu().numpy()


def _replay_device(db, sc, fields=True):
    import torch
    st = torch.cuda.Stream(device=torch.device("cuda", 0))
    out = []
    for op in sc.ops:
        if op[0] in ("loop", "reloc"):
            out.append(_detect_device(db, sc.K, op, st, fields))
        else:
            KS.replay(db, [op])
    return out


def _stateless_first_query(sc):
    """The scene's adds and covisibility lists before its first query as the arrays of orbfe_bow_db_detect (keyframe index =
    add order), or None when something else comes first."""
    adds, lists = [], {}
    for op in sc.ops:
        if op[0] == "add":
            adds.append(op)
        elif op[0] == "covis":
            lists.update(op[1])
        elif op[0] in ("loop", "reloc"):
            return adds, lists, op
        else:
            return None


@pytest.mark.parametrize("name", S.SCENE_NAMES)
def test_scene_host_and_device_forms_equal_the_oracle(gpu_required, voc, name):
    sc = S.scene(name)
    want = KS.replay(OracleDB(sc.K), sc.ops)
    dbs = [B.KeyFrameDatabase(voc, sc.K, sc.P) for _ in range(3)]
    try:
        _same(KS.replay(dbs[0], sc.ops), want, name + " host")
        _same(_replay_device(dbs[1], sc), want, name + " device")
        bare = _replay_device(dbs[2], sc, fields=False)      # d_words / d_score NULL: the same candidates
        assert len(bare) == len(want)
        for q, ((gc, _, _), (wc, _, _)) in enumerate(zip(bare, want)):
            assert np.array_equal(gc, wc), (name, q)
    finally:
        for db in dbs:
            db.close()
    first = _stateless_first_query(sc)
    if first is None:
        return
    adds, lists, op = first
    slot_of = [a[1] for a in adds]
    index_of = {s: k for k, s in enumerate(slot_of)}
    kf_ptr = np.cumsum([0] + [len(a[2]) for a in adds]).astype(np.int32)
    cov = [[index_of[x] for x in lists.get(s, [])] for s in slot_of]
    cp = np.cumsum([0] + [len(c) for c in cov]).astype(np.int32)
    mode = 0 if op[0] == "loop" else 1
    connected = np.zeros(len(adds), np.uint8)
    if mode == 0:
        connected[[index_of[c] for c in op[3]]] = 1
    m = fe.ORBmatcher(0.75, True)
    try:
        cand, common, score = B.db_detect(m, mode, op[1], op[2], kf_ptr, np.concatenate([a[2] for a in adds]),
                                          np.concatenate([a[3] for a in adds]), connected, cp, np.array(sum(cov, []) or [0], np.int32),
                                          op[4] if mode == 0 else 0.0)
    finally:
        m.close()
    wc, ww, ws = want[0]
    assert [slot_of[k] for k in cand] == wc.tolist(), name
    assert np.array_equal(np.where(ww[slot_of] < 0, 0, ww[slot_of]), common), name
    scored = score != -1
    assert np.array_equal(score[scored].view(np.int32), ws[slot_of][scored].view(np.int32)), name


# ---- capacity of the device form ----------------------------------------------------------------------------------------------
def test_device_form_capacity(gpu_required, voc):
    import torch
    sc = S.sizes(2049)
    want = KS.replay(OracleDB(sc.K), sc.ops)[0][0]
    n = len(want)
    assert n >= 1100
    db = B.KeyFrameDatabase(voc, sc.K, sc.P)
    try:
        KS.replay(db, [op for op in sc.ops if op[0] == "add"])
        op = next(op for op in sc.ops if op[0] == "reloc")
        mode, qi, qv, _, _, _ = _query_args(op)
        st = torch.cuda.Stream(device=torch.device("cuda", 0))
        GUARD = -7
        for cap in (0, 1, 1023, 1024, n - 1, n, n + 1):
            d_cand = torch.full((n + 8,), GUARD, dtype=torch.int32, device="cuda")
            d_n = torch.full((1,), GUARD, dtype=torch.int32, device="cuda")
            torch.cuda.synchronize()
            db.detect_device(mode, len(op[1]), qi.data_ptr(), qv.data_ptr(), 0, 0, 0.0, cap, d_cand.data_ptr(), d_n.data_ptr(),
                             stream=st.cuda_stream)
            st.synchronize()
            got = d_cand.cpu().numpy()
            k = min(cap, n)
            assert int(d_n.item()) == n, cap
            assert np.array_equal(got[:k], want[:k]), cap
            assert np.all(got[k:] == GUARD), cap                 # nothing written at or after entry cap
        # the host form: ORBFE_ERR_CAPACITY with the number needed, for every cap below n
        L = B._bind_kfdb()
        qi_h, qv_h = np.ascontiguousarray(op[1], np.int32), np.ascontiguousarray(op[2], np.float64)
        for cap in (0, 1, 1023, 1024, n - 1):
            cand, nc = np.zeros(max(cap, 1), np.int32), C.c_int(-1)
            rc = L.orbfe_kfdb_detect(db.handle, 1, len(qi_h), B._p(qi_h), B._p(qv_h), 0, None, 0.0, cap, B._p(cand), C.byref(nc), None, None)
            assert rc == fe.ORBFE_ERR_CAPACITY and nc.value == n, (cap, rc, nc.value)
        cand, _, _ = db.detect(1, op[1], op[2], cap=n)
        assert np.array_equal(cand, want)
    finally:
        db.close()


def test_nq_limit(gpu_required, voc):
    """nq = 65535 is accepted by both forms (and equals the oracle in the nq_65535 scene); 65536 is refused by both."""
    import torch
    db = B.KeyFrameDatabase(voc, 2, 70000)
    try:
        ids = np.arange(S.NWORDS, dtype=np.int32)
        vals = np.full(S.NWORDS, S.QV)
        db.add(0, ids[:10], vals[:10])
        with pytest.raises(fe.OrbfeError) as e:
            db.detect(1, ids, vals)
        assert e.value.code == fe.ORBFE_ERR_ARG
        qi, qv = _dev(ids, np.int32), _dev(vals, np.float64)
        d_cand, d_n = _zeros(2, torch.int32), _zeros(1, torch.int32)
        torch.cuda.synchronize()
        for mode in (0, 1):
            with pytest.raises(fe.OrbfeError) as e:
                db.detect_device(mode, len(ids), qi.data_ptr(), qv.data_ptr(), 0, 0, 0.0, 2, d_cand.data_ptr(), d_n.data_ptr())
            assert e.value.code == fe.ORBFE_ERR_ARG
        cand, words, _ = db.detect(1, ids[:65535], vals[:65535])
        assert list(cand) == [0] and words[0] == 10
    finally:
        db.close()


def test_max_keyframes_2_to_the_24(gpu_required, voc):
    """2^24 slots (about 3 GB of per-slot device arrays): keyframes in slots 0, 2^23 and 2^24 - 1 with covisibility across
    them, both query modes, equal to the oracle on the same scene at K = 3 with the slots remapped."""
    sc = S.tiny(3)
    big = 1 << 24
    remap = {0: 0, 1: 1 << 23, 2: big - 1}
    mapped = []
    for op in sc.ops:
        if op[0] in ("add", "erase"):
            mapped.append((op[0], remap[op[1]]) + tuple(op[2:]))
        elif op[0] == "covis":
            mapped.append(("covis", {remap[k]: [remap[x] for x in v] for k, v in op[1].items()}))
        elif op[0] == "loop":
            mapped.append(("loop", op[1], op[2], [remap[c] for c in op[3]], op[4]))
        else:
            mapped.append(op)
    assert {"loop", "reloc", "covis", "erase"} <= {op[0] for op in sc.ops}
    want = KS.replay(OracleDB(3), sc.ops)
    db = B.KeyFrameDatabase(voc, big, 64)
    try:
        got = KS.replay(db, mapped)
    finally:
        db.close()
    slots = [remap[k] for k in range(3)]
    for q, ((gc, gw, gs), (wc, ww, ws)) in enumerate(zip(got, want)):
        assert gc.tolist() == [remap[c] for c in wc.tolist()], q
        assert np.array_equal(gw[slots], ww) and np.array_equal(gs[slots].view(np.int32), ws.view(np.int32)), q
        assert np.count_nonzero(gw != -1) == np.count_nonzero(ww != -1) and np.count_nonzero(gs != -1) == np.count_nonzero(ws != -1), q
    assert len(got) == len(want)


# ---- stream ordering ----------------------------------------------------------------------------------------------------------
def test_query_chain_on_eight_streams(gpu_required, voc):
    """Eight relocalisation queries, each on its own stream into its own buffers, behind a spin on the first stream; one
    synchronisation at the end.  Query k reads the mRelocScore query k-1 left, so any reordering changes the candidates."""
    import torch
    sc = S.stream_chain(8)
    want = KS.replay(OracleDB(sc.K), sc.ops)
    db = B.KeyFrameDatabase(voc, sc.K, sc.P)
    try:
        KS.replay(db, [op for op in sc.ops if op[0] not in ("loop", "reloc")])
        queries = [op for op in sc.ops if op[0] == "reloc"]
        args = [_query_args(op) for op in queries]
        outs = [(_zeros(sc.K, torch.int32), _zeros(1, torch.int32), _zeros(sc.K, torch.int32), _zeros(sc.K, torch.float32)) for _ in queries]
        streams = [torch.cuda.Stream(device=torch.device("cuda", 0)) for _ in queries]
        torch.cuda.synchronize()
        with torch.cuda.stream(streams[0]):
            torch.cuda._sleep(SPIN)
        for op, (mode, qi, qv, _, _, _), (dc, dn, dw, ds), st in zip(queries, args, outs, streams):
            db.detect_device(mode, len(op[1]), qi.data_ptr(), qv.data_ptr(), 0, 0, 0.0, sc.K, dc.data_ptr(), dn.data_ptr(), dw.data_ptr(),
                             ds.data_ptr(), st.cuda_stream)
        torch.cuda.synchronize()
        got = [(dc[:int(dn.item())].cpu().numpy(), dw.cpu().numpy(), ds.cpu().numpy()) for dc, dn, dw, ds in outs]
    finally:
        db.close()
    _same(got, want, "chain")


@pytest.mark.parametrize("kind", ["erase", "add", "covis", "clear"])
def test_host_call_waits_for_the_pending_query(gpu_required, voc, kind):
    """A query enqueued on stream A behind a spin, then at once a synchronous host call that would change the query's result
    had it run first: the query sees the database as it was before the call; the next query sees the call."""
    import torch
    sc = S.host_call(kind)
    want = KS.replay(OracleDB(sc.K), sc.ops)
    db = B.KeyFrameDatabase(voc, sc.K, sc.P)
    try:
        KS.replay(db, sc.ops[:sc.pending])
        op = sc.ops[sc.pending]
        mode, qi, qv, _, _, _ = _query_args(op)
        dc, dn, dw, ds = _zeros(sc.K, torch.int32), _zeros(1, torch.int32), _zeros(sc.K, torch.int32), _zeros(sc.K, torch.float32)
        A = torch.cuda.Stream(device=torch.device("cuda", 0))
        torch.cuda.synchronize()
        with torch.cuda.stream(A):
            torch.cuda._sleep(SPIN)
        db.detect_device(mode, len(op[1]), qi.data_ptr(), qv.data_ptr(), 0, 0, 0.0, sc.K, dc.data_ptr(), dn.data_ptr(), dw.data_ptr(),
                         ds.data_ptr(), A.cuda_stream)
        KS.replay(db, [sc.ops[sc.pending + 1]])          # the host call, with the query still pending
        A.synchronize()
        first = (dc[:int(dn.item())].cpu().numpy(), dw.cpu().numpy(), ds.cpu().numpy())
        got = [first] + KS.replay(db, sc.ops[sc.pending + 2:])
    finally:
        db.close()
    _same(got, want, kind)
    assert not np.array_equal(want[0][0], want[1][0])      # the call changes the result


def test_add_device_after_rows_written_behind_a_spin(gpu_required, voc):
    """BowVector rows copied into place on stream A behind a spin, then orbfe_kfdb_add_device(stream = A) at once: the
    keyframes added are the rows' final contents (the queries after equal the oracle's)."""
    import torch
    sc = S.sizes(1025)
    adds = [op for op in sc.ops if op[0] == "add"]
    assert all(op[0] == "add" for op in sc.ops[:len(adds)])
    cap = max(len(a[2]) for a in adds)
    ids = np.full((len(adds), cap), np.iinfo(np.int32).max, np.int32)
    vals = np.zeros((len(adds), cap))
    for r, a in enumerate(adds):
        ids[r, :len(a[2])], vals[r, :len(a[2])] = a[2], a[3]
    counts = np.array([len(a[2]) for a in adds], np.int32)
    src = (_dev(ids, np.int32), _dev(vals, np.float64), _dev(counts, np.int32))
    dst = tuple(torch.zeros_like(t) for t in src)
    want = KS.replay(OracleDB(sc.K), sc.ops)
    db = B.KeyFrameDatabase(voc, sc.K, sc.P)
    try:
        A = torch.cuda.Stream(device=torch.device("cuda", 0))
        torch.cuda.synchronize()
        with torch.cuda.stream(A):
            torch.cuda._sleep(SPIN)
            for d, s in zip(dst, src):
                d.copy_(s)
        db.add_device([a[1] for a in adds], np.arange(len(adds)), cap, dst[0].data_ptr(), dst[1].data_ptr(), dst[2].data_ptr(),
                      stream=A.cuda_stream)
        assert db.size() == (len(adds), int(counts.sum()))
        got = KS.replay(db, sc.ops[len(adds):])
    finally:
        db.close()
    _same(got, want, "add_device")
