"""GPU tests of the resident covisibility graph (include/orbfe_bow.h orbfe_covis_*): after every step of every scene of
tests/covis_scenes.py the device graph, read whole through orbfe_covis_lists_device (both lists, nbest 10, 20 and all), equals
the oracle that tests/test_oracle_covis.py pins to the reference's own KeyFrame.cc; a batch equals batches of one; bad input
and overflow leave the graph unchanged and are reported by sync; set_covisibles_device on an export answers queries as the
host set_covisibles on the oracle's lists; and extraction -> BowVectors -> update_connections_device -> lists_device ->
bow_min_score_device + set_covisibles_device + detect_batch_device (loop mode) equals the same chain fed the oracle's lists
from the host."""
import numpy as np
import pytest

import orb_slam_b200 as fe
from oracle.covis import CovisOracle
from orb_slam_b200 import bow as B

import covis_scenes as S

pytestmark = pytest.mark.gpu


def _torch():
    import torch
    return torch, torch.device("cuda", 0)


def _dev(a, dt=np.int32):
    torch, dev = _torch()
    return torch.from_numpy(np.ascontiguousarray(a, dt)).to(dev)


def export(g, slots, which, nbest):
    """(ptr, list, weights) of lists_device as host arrays"""
    torch, dev = _torch()
    n = len(slots)
    lim = min(nbest, g.max_connections) if which == 0 and nbest > 0 else g.max_connections
    d_ptr = torch.full((n + 1,), -7, dtype=torch.int32, device=dev)
    d_list = torch.full((max(n * lim, 1),), -7, dtype=torch.int32, device=dev)
    d_w = torch.full((max(n * lim, 1),), -7, dtype=torch.int32, device=dev)
    g.lists_device(which, slots, nbest, d_ptr.data_ptr(), d_list.data_ptr(), d_w.data_ptr())
    g.sync()
    ptr = d_ptr.cpu().numpy()
    return ptr, d_list.cpu().numpy()[:ptr[-1]], d_w.cpu().numpy()[:ptr[-1]]


def state(g, K):
    """the whole graph as exported: both lists with weights, and the best-10 / best-20 rows"""
    slots = np.arange(K)
    return [tuple(a.tolist() for a in export(g, slots, which, nb)) for which, nb in ((0, -1), (0, 10), (0, 20), (1, 0))]


def oracle_state(orc, K):
    out = []
    dead = lambda s: s if orc.live(s) else -1
    for which, nb in ((0, -1), (0, 10), (0, 20), (1, 0)):
        ptr, lst, ws = [0], [], []
        for s in range(K):
            sl, w = orc.ordered(s) if which == 0 else orc.weights(s)
            if which == 0 and nb > 0:
                sl, w = sl[:nb], w[:nb]
            lst += [dead(x) for x in sl]
            ws += w
            ptr.append(len(lst))
        out.append((ptr, lst, ws))
    return out


class Run:
    """A scene on the device graph (batches as given, or cut into batches of one) and on the oracle."""

    def __init__(self, scene, single=False, max_batch=64, max_connections=None):
        self.scene, self.single = scene, single
        self.K = scene.nkf
        self.slot_of = scene.slots()
        self.model = S.Model(scene)
        self.g = B.CovisibilityGraph(self.K, max_connections or scene.max_connections, max_batch)
        self.orc = CovisOracle(self.K)
        self._dv = None

    def close(self):
        self.g.close()
        self.orc.close()

    def inputs(self):
        kf_mp, counts, gp, obs = self.model.inputs(self.slot_of, self.K)
        if self._dv is None or self._dv[0] != self.model.version:
            self._dv = (self.model.version, [_dev(kf_mp), _dev(counts), _dev(gp), _dev(obs if len(obs) else [0])], (kf_mp, counts, gp, obs))
        return self._dv[1], self._dv[2]

    def update_device(self, slots, d=None, npoints=None, nobs=None):
        torch, dev = _torch()
        (d_mp, d_cnt, d_gp, d_obs), (_, _, gp, obs) = self.inputs()
        if d is not None:
            d_mp, d_cnt, d_gp, d_obs = d
        d_par = torch.full((len(slots),), -9, dtype=torch.int32, device=dev)
        self.g.update_connections_device(slots, d_mp.data_ptr(), d_cnt.data_ptr(), self.K, self.scene.cap, d_gp.data_ptr(), d_obs.data_ptr(),
                                         len(gp) - 1 if npoints is None else npoints, len(obs) if nobs is None else nobs, d_par.data_ptr())
        return d_par

    def step(self, step):
        self.model.apply(step)
        op = step[0]
        if op == "kf":
            k = len(self.model.nfeat) - 1
            s = int(self.slot_of[k])
            self.g.add([s], [k], [k])
            self.orc.add(s, k, k)
        elif op == "update":
            slots = [int(self.slot_of[k]) for k in step[1]]
            _, (kf_mp, counts, gp, obs) = self.inputs()
            want = self.orc.replay(slots, kf_mp, counts, self.scene.cap, gp, obs)
            groups = [[s] for s in slots] if self.single else [slots[i:i + self.g.max_batch] for i in range(0, len(slots), self.g.max_batch)]
            got = []
            for grp in groups:
                d_par = self.update_device(grp)
                self.g.sync()
                got += d_par.cpu().numpy().tolist()
            assert got == want, (self.scene.name, step)
        elif op == "erase_kf":
            s = int(self.slot_of[step[1]])
            self.g.erase(s)
            self.orc.erase(s)

    def check(self, where):
        assert state(self.g, self.K) == oracle_state(self.orc, self.K), where


SMALL = S.small_scenes()


@pytest.mark.parametrize("scene", SMALL, ids=lambda s: s.name)
def test_device_equals_oracle_after_every_step(gpu_required, scene):
    r = Run(scene)
    try:
        for t, step in enumerate(scene.steps):
            r.step(step)
            r.check((scene.name, t, step[0]))
    finally:
        r.close()


@pytest.fixture(scope="module")
def large():
    return S.scene_large()


def test_large_map_batches_of_64(gpu_required, large):
    """2000 keyframes x 2000 features, ~8 observations per point: batches of 64 equal the oracle after every batch"""
    r = Run(large, max_batch=64)
    try:
        for t, step in enumerate(large.steps):
            r.step(step)
            if step[0] == "update":
                r.check(("large", t))
    finally:
        r.close()


@pytest.mark.parametrize("name", ["batch30", "large"])
def test_batch_equals_batches_of_one(gpu_required, large, name):
    scene = large if name == "large" else S.scene_batch30()
    a, b = Run(scene, max_batch=64), Run(scene, single=True, max_batch=64)
    try:
        for step in scene.steps:
            a.step(step)
            b.step(step)
        assert state(a.g, a.K) == state(b.g, b.K) == oracle_state(a.orc, a.K)
    finally:
        a.close()
        b.close()


def _snapshot(r):
    return state(r.g, r.K)


def test_capacity_exact_and_one_over(gpu_required):
    scene, hub, hub2 = S.scene_capacity(6)
    r = Run(scene)
    try:
        for step in scene.steps:
            r.step(step)
        sh, sh2 = int(r.slot_of[hub]), int(r.slot_of[hub2])
        r.update_device([sh])          # exactly max_connections neighbours
        r.g.sync()
        ptr, lst, _ = export(r.g, [sh], 1, 0)
        assert ptr[-1] == 6
        before = _snapshot(r)
        d_par = r.update_device([sh2])   # one more than max_connections
        with pytest.raises(fe.OrbfeError) as e:
            r.g.sync()
        assert e.value.code == fe.ORBFE_ERR_CAPACITY
        assert d_par.cpu().numpy().tolist() == [-1]
        assert _snapshot(r) == before
        r.g.sync()   # reported once
    finally:
        r.close()


def test_capacity_of_a_target_filled_by_an_event(gpu_required):
    """a neighbour whose map is full: the AddConnection another keyframe's update sends it would be one entry too many"""
    s = S.Scene("target_full", 64, seed=13, max_connections=2)
    T, A, Bk, E = s.kf(), s.kf(), s.kf(), s.kf()
    f = [0] * 4
    f[T], f[A] = S._share(s, T, A, 20, f[T], f[A])
    f[T], f[Bk] = S._share(s, T, Bk, 20, f[T], f[Bk])
    s.update([T])                                   # T: {A, B}, exactly max_connections
    f[T], f[E] = S._share(s, T, E, 20, f[T], f[E])  # E's own counter is {T}: one entry
    r = Run(s)
    try:
        for step in s.steps:
            r.step(step)
        r.check("before")
        before = _snapshot(r)
        d_par = r.update_device([int(r.slot_of[E])])
        with pytest.raises(fe.OrbfeError) as e:
            r.g.sync()
        assert e.value.code == fe.ORBFE_ERR_CAPACITY
        assert d_par.cpu().numpy().tolist() == [-1]
        assert _snapshot(r) == before
    finally:
        r.close()


def test_bad_input_rejects_the_batch(gpu_required):
    scene = S.scene_culling()
    r = Run(scene)
    torch, dev = _torch()
    try:
        for step in scene.steps:
            r.step(step)
        before = _snapshot(r)
        (d_mp, d_cnt, d_gp, d_obs), (kf_mp, counts, gp, obs) = r.inputs()
        live = [int(r.slot_of[k]) for k in range(scene.nkf) if not r.model.kf_bad[k]]
        A = int(r.slot_of[0])
        dead = int(r.slot_of[1])
        cases = []
        cases.append(("point index >= npoints", None, dict(npoints=int(kf_mp.max()))))
        p = int(kf_mp[(kf_mp >= 0) & (np.repeat(np.arange(r.K), scene.cap) == A)][0])   # a point A sees
        bad_gp = gp.copy()
        bad_gp[p] = bad_gp[p + 1] + 1
        cases.append(("group pointer", (d_mp, d_cnt, _dev(bad_gp), d_obs), {}))
        o2 = obs.copy()
        o2[gp[p]] = r.K * scene.cap       # frame >= nframes
        cases.append(("frame out of range", (d_mp, d_cnt, d_gp, _dev(o2)), {}))
        o3 = obs.copy()
        o3[gp[p]] = dead * scene.cap      # a retired slot
        cases.append(("retired observer", (d_mp, d_cnt, d_gp, _dev(o3)), {}))
        c2 = counts.copy()
        c2[A] = scene.cap + 1
        cases.append(("count > cap", (d_mp, _dev(c2), d_gp, d_obs), {}))
        for name, d, kw in cases:
            d_par = r.update_device(live, d=d, **kw)
            with pytest.raises(fe.OrbfeError) as e:
                r.g.sync()
            assert e.value.code == fe.ORBFE_ERR_ARG, name
            assert d_par.cpu().numpy().tolist() == [-1] * len(live), name
            assert _snapshot(r) == before, name
        r.g.sync()   # the error was reported once
        # the stale entry keeps the retired slot from being re-added; once A's own update drops it, the slot is free
        with pytest.raises(fe.OrbfeError):
            r.g.add([dead], [99], [99])
        r.update_device([A])
        r.g.sync()
        r.g.add([dead], [99], [99])
    finally:
        r.close()


def _db_pair(voc, K, rng, erased):
    dbs = [B.KeyFrameDatabase(voc, K, K * 64), B.KeyFrameDatabase(voc, K, K * 64)]
    bows = []
    for s in range(K):
        ids = np.sort(rng.choice(200, size=40, replace=False)).astype(np.int32)
        vals = rng.random(40)
        vals /= vals.sum()
        bows.append((ids, vals))
        for db in dbs:
            db.add(s, ids, vals)
    for s in erased:
        for db in dbs:
            db.erase(s)
    return dbs, bows


def test_set_covisibles_device_equals_host_lists(gpu_required):
    """an export with a stale -1 inside the first 10 answers queries as the host form fed the oracle's lists"""
    from test_gpu_kfdb import flat_vocabulary
    scene = S.scene_culling()
    r = Run(scene)
    torch, dev = _torch()
    V = B.Vocabulary(flat_vocabulary(200))
    try:
        for step in scene.steps:
            r.step(step)
        K = r.K
        dead = [s for s in range(K) if not r.orc.live(s)]
        A = int(r.slot_of[0])
        assert -1 in export(r.g, [A], 0, 10)[1].tolist()          # the stale entry is exported inside the first 10
        host, dv = _db_pair(V, K, np.random.default_rng(3), dead)[0]
        live = [s for s in range(K) if r.orc.live(s)]
        host.set_covisibles({s: r.orc.ordered(s)[0][:10] for s in live})
        ptr, lst, _ = export(r.g, live, 0, -1)
        d_ptr, d_lst = _dev(ptr), _dev(lst if len(lst) else [0])   # alive until the enqueued copy has run
        dv.set_covisibles_device(live, d_ptr.data_ptr(), d_lst.data_ptr())
        rng = np.random.default_rng(4)
        for q in range(6):
            ids = np.sort(rng.choice(200, size=60, replace=False)).astype(np.int32)
            vals = rng.random(60)
            for mode in (0, 1):
                conn = r.orc.weights(live[q % len(live)])[0] if mode == 0 else ()
                a = host.detect(mode, ids, vals, connected=conn, min_score=0.001)
                b = dv.detect(mode, ids, vals, connected=conn, min_score=0.001)
                assert np.array_equal(a[0], b[0]) and np.array_equal(a[1], b[1]) and np.array_equal(a[2].view(np.int32), b[2].view(np.int32))
        host.close()
        dv.close()
    finally:
        V.close()
        r.close()


def test_chain_extract_update_lists_min_score_detect(gpu_required):
    """frame store -> update_connections_device -> lists_device -> bow_min_score_device + set_covisibles_device +
    detect_batch_device (loop mode), with no index upload between the calls, equals the chain fed the oracle's lists"""
    torch, dev = _torch()
    from orb_slam_b200.synth import random_vocabulary, shifted_frame, textured_frame
    W, H, NF, levelsup = 640, 480, 1000, 3
    NKF, NQ = 16, 4
    bases = [textured_frame(W, H, seed=21), textured_frame(W, H, seed=22)]
    frames = np.stack([shifted_frame(bases[i % 2], 2 * i - 16, 1 - i // 4, seed=60 + i) for i in range(NKF)])
    V = B.Vocabulary(random_vocabulary(10, 4, seed=6))
    ex = fe.ORBextractor(NF, 1.2, 8)
    s = torch.cuda.Stream(device=dev)
    z = lambda *shape: torch.zeros(shape, dtype=torch.int32, device=dev)
    d_frames = torch.from_numpy(frames).to(dev)
    d_kps, d_desc = torch.zeros((NKF, NF, 28), dtype=torch.uint8, device=dev), torch.zeros((NKF, NF, 32), dtype=torch.uint8, device=dev)
    d_cnt, d_leaf, d_node = z(NKF), z(NKF * NF), z(NKF * NF)
    d_bid, d_bval, d_bn = z(NKF, NF), torch.zeros((NKF, NF), dtype=torch.float64, device=dev), z(NKF)
    torch.cuda.synchronize()
    ex.extract_batch_device(d_frames.data_ptr(), W, H, W, W * H, NKF, d_kps.data_ptr(), d_desc.data_ptr(), d_cnt.data_ptr(), s.cuda_stream)
    V.descend_device(d_desc.data_ptr(), NKF * NF, levelsup, d_leaf.data_ptr(), d_node.data_ptr(), s.cuda_stream)
    B.bow_vector_device(V, NKF, d_leaf.data_ptr(), d_cnt.data_ptr(), NF, d_bid.data_ptr(), d_bval.data_ptr(), d_bn.data_ptr(), s.cuda_stream)
    s.synchronize()
    counts = d_cnt.cpu().numpy()
    assert counts.min() >= 400
    # observations: keyframe f sees points shared with f-1 .. f-3 at its first 400 features; slot = frame row, key = row
    rng = np.random.default_rng(5)
    kf_mp = np.full((NKF, NF), -1, np.int32)
    obs_of = []
    free = np.zeros(NKF, np.int64)
    for f in range(1, NKF):
        for back in (1, 2, 3):
            if f - back < 0:
                continue
            for _ in range(int(rng.integers(5, 40))):
                if free[f] >= 400 or free[f - back] >= 400:
                    break
                m = len(obs_of)
                obs_of.append([(f - back, int(free[f - back])), (f, int(free[f]))])
                kf_mp[f - back, free[f - back]] = m
                kf_mp[f, free[f]] = m
                free[f - back] += 1
                free[f] += 1
    gp = np.zeros(len(obs_of) + 1, np.int32)
    gp[1:] = np.cumsum([len(o) for o in obs_of])
    obs = np.array([k * NF + i for o in obs_of for k, i in sorted(o)], np.int32)
    g = B.CovisibilityGraph(NKF, 64, 64)
    orc = CovisOracle(NKF)
    slots = list(range(NKF))
    g.add(slots, slots, slots)
    for k in slots:
        orc.add(k, k, k)
    d_mp, d_gp, d_obs = _dev(kf_mp), _dev(gp), _dev(obs)
    order = list(range(1, NKF)) + [0]
    g.update_connections_device(order, d_mp.data_ptr(), d_cnt.data_ptr(), NKF, NF, d_gp.data_ptr(), d_obs.data_ptr(), len(obs_of), len(obs),
                                stream=s.cuda_stream)
    orc.replay(order, kf_mp.ravel(), counts, NF, gp, obs)
    queries = list(range(NKF - NQ, NKF))
    db_slots = np.arange(0, NKF - NQ)
    dbs = [B.KeyFrameDatabase(V, NKF, NKF * NF, NQ), B.KeyFrameDatabase(V, NKF, NKF * NF, NQ)]
    res = []
    try:
        for db in dbs:
            db.add_device(db_slots, db_slots, NF, d_bid.data_ptr(), d_bval.data_ptr(), d_bn.data_ptr(), stream=s.cuda_stream)
        # device chain: every index list comes from lists_device
        d_cptr, d_crow = z(NQ + 1), z(NQ * 64)
        d_nptr, d_conn = z(NQ + 1), z(NQ * 64)
        d_bptr, d_best = z(NKF + 1), z(NKF * 10)
        g.lists_device(0, queries, 0, d_cptr.data_ptr(), d_crow.data_ptr(), stream=s.cuda_stream)
        g.lists_device(1, queries, 0, d_nptr.data_ptr(), d_conn.data_ptr(), stream=s.cuda_stream)
        g.lists_device(0, slots, 10, d_bptr.data_ptr(), d_best.data_ptr(), stream=s.cuda_stream)
        d_q = _dev(queries)
        torch.cuda.synchronize()
        chains = [(dbs[0], d_cptr, d_crow, d_nptr, d_conn, True)]
        # host chain: the oracle's lists uploaded
        cov = [orc.ordered(q)[0] for q in queries]
        con = [orc.weights(q)[0] for q in queries]
        hp = lambda L: np.concatenate([[0], np.cumsum([len(x) for x in L])]).astype(np.int32)
        hl = lambda L: np.array(sum(L, []) or [0], np.int32)
        chains.append((dbs[1], _dev(hp(cov)), _dev(hl(cov)), _dev(hp(con)), _dev(hl(con)), False))
        dbs[1].set_covisibles({k: orc.ordered(k)[0][:10] for k in slots})
        for db, cptr, crow, nptr, conn, device in chains:
            if device:
                db.set_covisibles_device(slots, d_bptr.data_ptr(), d_best.data_ptr(), stream=s.cuda_stream)
            d_min = torch.zeros(NQ, dtype=torch.float32, device=dev)
            B.min_score_device(V, NQ, NKF, NF, d_bid.data_ptr(), d_bval.data_ptr(), d_bn.data_ptr(), d_q.data_ptr(), cptr.data_ptr(),
                               crow.data_ptr(), 0, d_min.data_ptr(), s.cuda_stream)
            d_cand, d_nc = z(NQ * NKF), z(NQ)
            d_words, d_score = z(NQ * NKF), torch.zeros(NQ * NKF, dtype=torch.float32, device=dev)
            qrows = d_bid[NKF - NQ:].contiguous(), d_bval[NKF - NQ:].contiguous()
            db.detect_batch_device(0, NQ, NF, qrows[0].data_ptr(), qrows[1].data_ptr(), nptr.data_ptr(), conn.data_ptr(), d_min.data_ptr(), NKF,
                                   d_cand.data_ptr(), d_nc.data_ptr(), d_words.data_ptr(), d_score.data_ptr(), stream=s.cuda_stream)
            s.synchronize()
            res.append((d_min.cpu().numpy(), d_nc.cpu().numpy(), d_cand.cpu().numpy(), d_words.cpu().numpy(), d_score.cpu().numpy()))
        g.sync()
        (m0, n0, c0, w0, s0), (m1, n1, c1, w1, s1) = res
        assert np.array_equal(m0.view(np.int32), m1.view(np.int32))
        assert np.array_equal(n0, n1) and np.array_equal(w0, w1) and np.array_equal(s0.view(np.int32), s1.view(np.int32))
        for b in range(NQ):
            assert np.array_equal(c0[b * NKF:b * NKF + n0[b]], c1[b * NKF:b * NKF + n1[b]])
        assert (m0 < 1).all()   # every query had connected keyframes that share words
    finally:
        for db in dbs:
            db.close()
        g.close()
        orc.close()
        ex.close()
        V.close()
