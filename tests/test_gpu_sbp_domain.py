"""The scenes of sbp_domain_scenes.py through every entry of the fused projection matcher that can express them, bit for
bit against the oracle (which test_oracle_sbp_domain.py holds to the sequential model): reservation chains past the
48-round fallback, displacement cascades, MODE-2 re-assignment and the rotation histogram on its boundaries.  Explicit
windows go through orbfe_guided_search (hist_mode 0 and 1) and orbfe_guided_search_device (several jobs per launch); the
same scenes realised as projections (identity pose, fx = fy = 1, cx = cy = 0: the projection of (u, v, 1) is exactly
(u, v)) or keypoint windows go through orbfe_window_search, orbfe_search_local_points, orbfe_search_by_projection_f1f2,
orbfe_search_by_projection_kf, orbfe_search_by_projection_frames / _device and orbfe_search_for_initialization / _device.
Every test runs with the candidate entries in shared memory and in the global scratch."""
import os

import numpy as np
import pytest

import oracle as O
import orb_slam_b200 as fe
import sbp_domain_scenes as S
from orb_slam_b200 import matching as M

pytestmark = pytest.mark.gpu

W, H = S.W, S.H
WIN = int(S.R)


@pytest.fixture(params=[0, 1], ids=["smem-entries", "global-scratch"], autouse=True)
def placement(request):
    if request.param:
        os.environ["ORBFE_SBP_FORCE_SCRATCH"] = "1"
    yield request.param
    os.environ.pop("ORBFE_SBP_FORCE_SCRATCH", None)


_cache = {}


def scene(name):
    if name not in _cache:
        make = {"chains-rule1": lambda: S.chains_scene(1), "chains-rule2": lambda: S.chains_scene(2),
                "tails-rule1": lambda: S.tails_scene(1), "tails-rule2": lambda: S.tails_scene(2), "ties-rule1": S.tie_tails_scene,
                "star-1000": lambda: S.star_scene(1000), "ladders": S.ladder_scene, "init": S.init_scene}
        if name in make:
            _cache[name] = make[name]()
        else:
            _cache[name] = next(s for s in S.hist_scenes() if s.name == name)
    return _cache[name]


def _views(sc):
    return M.FrameView(sc.kps, sc.desc, W, H), O.OracleFrame(sc.kps, sc.desc, W, H)


HIST = ["max2-at", "max3-at", "max2-below", "max3-below", "max-ties", "angles"]
GUIDED = ["chains-rule1", "chains-rule2", "tails-rule1", "tails-rule2", "ties-rule1", "star-1000", "ladders"] + HIST


@pytest.mark.parametrize("hist", [0, 1])
@pytest.mark.parametrize("name", GUIDED)
def test_guided_search(gpu_required, name, hist):
    sc = scene(name)
    v, o = _views(sc)
    m = fe.ORBmatcher(sc.nnratio, False)
    args = (sc.qu, sc.qv, sc.qr, sc.qlo, sc.qhi, sc.qdesc, sc.qangle, sc.rule)
    n, so = M.guided_search(m, v, *args, sc.th_dist, hist, slot_owner=sc.slot_owner())
    n_o, so_o = O.guided_search(o, *args, sc.nnratio, sc.th_dist, hist, slot_owner=sc.slot_owner())
    m.close()
    assert n == n_o and np.array_equal(so, so_o)
    if hist == sc.hist:
        assert n == S.sequential(sc)[0]


# ---- several jobs in one device launch ----

def _job_scenes(rule):
    """Chain depths 0 (no queries), 48, 49, 200 (blocked, so every query matches) and a 49-deep free chain with a 65-entry
    tail; rule 0: ladders of the same depths and a 256-query star."""
    out = []
    for depth in (0, 48, 49, 200):
        b = S.Builder(10 + depth)
        sc = S.Scene("job", rule)
        if depth:
            (S.add_ladder(b, depth) if rule == 0 else S.add_chain(b, depth, True, rule))
        else:
            b.slot(10.0, 20.0)
        out.append(b.build(sc) if depth else _empty(b, sc))
    if rule == 0:
        out.append(S.star_scene(256))
    else:
        b = S.Builder(99)
        S.add_chain(b, 49, False, rule, tail=65)
        out.append(b.build(S.Scene("job", rule)))
    return out


def _empty(b, sc):
    sc.kps = np.zeros(1, S.KP_DTYPE)
    sc.kps["x"], sc.kps["y"] = 10.0, 20.0
    sc.desc = np.zeros((1, 32), np.uint8)
    sc.qu = sc.qv = sc.qr = sc.qangle = np.zeros(0, np.float32)
    sc.qlo = sc.qhi = np.zeros(0, np.int32)
    sc.qdesc = np.zeros((0, 32), np.uint8)
    sc.occ, sc.lists, sc.dist = np.zeros(1, bool), [], []
    return sc


@pytest.mark.parametrize("ori", [False, True])
@pytest.mark.parametrize("rule", [0, 1, 2])
def test_guided_search_device_jobs(gpu_required, rule, ori):
    import torch
    jobs = _job_scenes(rule)
    cap = 1024
    nj = len(jobs)
    kps = np.zeros((nj, cap), fe.KP_DTYPE)
    desc = np.zeros((nj, cap, 32), np.uint8)
    pre = np.full((nj, cap), -1, np.int32)
    counts = np.array([sc.n for sc in jobs], np.int32)
    for j, sc in enumerate(jobs):
        kps[j, :sc.n], desc[j, :sc.n], pre[j, :sc.n] = sc.kps, sc.desc, sc.slot_owner()
    cat = lambda f, t: np.ascontiguousarray(np.concatenate([getattr(sc, f) for sc in jobs]).astype(t))
    Q = [cat("qu", np.float32), cat("qv", np.float32), cat("qr", np.float32), cat("qlo", np.int32), cat("qhi", np.int32),
         np.ascontiguousarray(np.concatenate([sc.qdesc for sc in jobs])), cat("qangle", np.float32)]
    qcnt = np.array([sc.nq for sc in jobs], np.int32)
    qbase = np.concatenate([[0], np.cumsum(qcnt)[:-1]]).astype(np.int32)
    dev = torch.device("cuda", 0)
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev)
    d_kps, d_desc, d_cnt, d_fi = t(kps.view(np.uint8).reshape(nj, cap, 28)), t(desc), t(counts), t(np.arange(nj, dtype=np.int32))
    d_q = [t(x) for x in Q]
    d_qb, d_qc = t(qbase), t(qcnt)
    d_so, d_nm = t(pre), torch.zeros(nj, dtype=torch.int32, device=dev)
    m = fe.ORBmatcher(0.75, ori)
    M.guided_search_device(m, nj, d_kps.data_ptr(), d_desc.data_ptr(), d_cnt.data_ptr(), cap, d_fi.data_ptr(),
                           *[x.data_ptr() for x in d_q], d_qb.data_ptr(), d_qc.data_ptr(), max(int(qcnt.max()), 1), W, H,
                           rule, S.TH_HIGH, d_so.data_ptr(), d_nm.data_ptr())
    m.sync()
    m.close()
    so, nm = d_so.cpu().numpy(), d_nm.cpu().numpy()
    for j, sc in enumerate(jobs):
        n_o, so_o = O.guided_search(O.OracleFrame(sc.kps, sc.desc, W, H), sc.qu, sc.qv, sc.qr, sc.qlo, sc.qhi, sc.qdesc, sc.qangle,
                                    rule, 0.75, S.TH_HIGH, int(ori), slot_owner=sc.slot_owner())
        assert nm[j] == n_o and np.array_equal(so[j, :sc.n], so_o), j


# ---- the same scenes realised through the routine-level entries ----

_last_frame, _world, T_ID = S.f1_keypoints, S.world_points, S.T_ID


def _rule0_scenes():
    return ["ladders", "star-1000"] + HIST


@pytest.mark.parametrize("ori", [False, True])
@pytest.mark.parametrize("name", _rule0_scenes())
def test_search_by_projection_frames(gpu_required, name, ori):
    """SearchByProjection(Frame, Frame, th = 6) with the Last features at the window centres: rule 0 at TH_HIGH."""
    import torch
    sc = scene(name)
    lk = _last_frame(sc)
    has, outl, world = np.ones(sc.nq, np.uint8), np.zeros(sc.nq, np.uint8), _world(sc)
    m = fe.ORBmatcher(0.9, ori)
    cur, last = M.FrameView(sc.kps, sc.desc, W, H), M.FrameView(lk, sc.qdesc, W, H)
    nm, mp = M.search_by_projection_frames(m, [cur], [last], [has], [outl], [world], [T_ID], 1.0, 1.0, 0.0, 0.0, float(WIN),
                                           cur_mp=[sc.slot_owner()])
    n_o, mp_o = O.search_by_projection_ff(O.OracleFrame(sc.kps, sc.desc, W, H), O.OracleFrame(lk, sc.qdesc, W, H), has, outl, world,
                                          T_ID, 1.0, 1.0, 0.0, 0.0, float(WIN), check_orientation=ori, cur_mp=sc.slot_owner())
    assert nm[0] == n_o and np.array_equal(mp[0], mp_o)
    # device form: Current = frame 0, Last = frame 1 of a two-frame store.  Its scratch holds 64 candidate entries per
    # feature of cap and it does not relaunch (the host form does): the 1000-query star's million entries stay on the host
    # form here and reach the device form as a 256-query star in test_search_by_projection_device_jobs
    cap = max(sc.n, sc.nq)
    if sum(len(l) for l in sc.lists) > 64 * cap:
        assert name == "star-1000"
        return
    kps = np.zeros((2, cap), fe.KP_DTYPE)
    desc = np.zeros((2, cap, 32), np.uint8)
    kps[0, :sc.n], desc[0, :sc.n], kps[1, :sc.nq], desc[1, :sc.nq] = sc.kps, sc.desc, lk, sc.qdesc
    w = np.zeros((2, cap, 3), np.float32)
    w[1, :sc.nq] = world
    fl = np.zeros((2, cap), np.uint8)
    fl[1, :sc.nq] = 1
    pre = np.full((1, cap), -1, np.int32)
    pre[0, :sc.n] = sc.slot_owner()
    dev = torch.device("cuda", 0)
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev)
    d_mp, d_nm = t(pre), torch.zeros(1, dtype=torch.int32, device=dev)
    d = [t(kps.view(np.uint8).reshape(2, cap, 28)), t(desc), t(np.array([sc.n, sc.nq], np.int32)), t(np.array([0], np.int32)),
         t(np.array([1], np.int32)), t(w), t(fl), t(T_ID.reshape(1, 12))]
    M.search_by_projection_device(m, 1, d[0].data_ptr(), d[1].data_ptr(), d[2].data_ptr(), cap, d[3].data_ptr(), d[4].data_ptr(),
                                  d[5].data_ptr(), d[6].data_ptr(), d[7].data_ptr(), W, H, 1.2, 8, 1.0, 1.0, 0.0, 0.0, float(WIN),
                                  d_mp.data_ptr(), d_nm.data_ptr())
    m.sync()
    m.close()
    assert int(d_nm.cpu()[0]) == n_o and np.array_equal(d_mp.cpu().numpy()[0, :sc.n], mp_o)


@pytest.mark.parametrize("ori", [False, True])
def test_search_by_projection_device_jobs(gpu_required, ori):
    """orbfe_search_by_projection_device with several pairs in one launch: ladders of depth 0 (no Last features), 48, 49
    and 200 and a 256-query star, each pair = (the scene's slots, a Last frame at its window centres)."""
    import torch
    jobs = _job_scenes(0)
    nj, cap = len(jobs), 1024
    kps = np.zeros((2 * nj, cap), fe.KP_DTYPE)
    desc = np.zeros((2 * nj, cap, 32), np.uint8)
    world = np.zeros((2 * nj, cap, 3), np.float32)
    flags = np.zeros((2 * nj, cap), np.uint8)
    counts = np.zeros(2 * nj, np.int32)
    pre = np.full((nj, cap), -1, np.int32)
    for j, sc in enumerate(jobs):
        assert sum(len(l) for l in sc.lists) <= 64 * cap
        kps[2 * j, :sc.n], desc[2 * j, :sc.n], counts[2 * j], pre[j, :sc.n] = sc.kps, sc.desc, sc.n, sc.slot_owner()
        kps[2 * j + 1, :sc.nq], desc[2 * j + 1, :sc.nq], counts[2 * j + 1] = _last_frame(sc), sc.qdesc, sc.nq
        world[2 * j + 1, :sc.nq], flags[2 * j + 1, :sc.nq] = _world(sc), 1
    dev = torch.device("cuda", 0)
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev)
    d = [t(kps.view(np.uint8).reshape(2 * nj, cap, 28)), t(desc), t(counts), t(2 * np.arange(nj, dtype=np.int32)),
         t(2 * np.arange(nj, dtype=np.int32) + 1), t(world), t(flags), t(np.tile(T_ID.reshape(1, 12), (nj, 1)))]
    d_mp, d_nm = t(pre), torch.zeros(nj, dtype=torch.int32, device=dev)
    m = fe.ORBmatcher(0.9, ori)
    M.search_by_projection_device(m, nj, *[x.data_ptr() for x in d[:3]], cap, *[x.data_ptr() for x in d[3:]], W, H, 1.2, 8,
                                  1.0, 1.0, 0.0, 0.0, float(WIN), d_mp.data_ptr(), d_nm.data_ptr())
    m.sync()
    m.close()
    mp, nm = d_mp.cpu().numpy(), d_nm.cpu().numpy()
    for j, sc in enumerate(jobs):
        has, outl = np.ones(sc.nq, np.uint8), np.zeros(sc.nq, np.uint8)
        n_o, mp_o = O.search_by_projection_ff(O.OracleFrame(sc.kps, sc.desc, W, H), O.OracleFrame(_last_frame(sc), sc.qdesc, W, H),
                                              has, outl, _world(sc), T_ID, 1.0, 1.0, 0.0, 0.0, float(WIN), check_orientation=ori,
                                              cur_mp=sc.slot_owner())
        assert nm[j] == n_o and np.array_equal(mp[j, :sc.n], mp_o), j
    assert nm.sum() == 48 + 49 + 200 + 256


@pytest.mark.parametrize("ori", [False, True])
@pytest.mark.parametrize("name", _rule0_scenes())
def test_search_by_projection_kf(gpu_required, name, ori):
    """SearchByProjection(Frame, KeyFrame, th = 6, ORBdist = 100): min_dist 1e9 predicts level 0 (octaves -1..1)."""
    sc = scene(name)
    valid, world, md = np.ones(sc.nq, np.uint8), _world(sc), np.full(sc.nq, 1e9, np.float32)
    m = fe.ORBmatcher(0.9, ori)
    n, mp = M.search_by_projection_kf(m, M.FrameView(sc.kps, sc.desc, W, H), valid, world, md, sc.qdesc, sc.qangle, T_ID,
                                      1.0, 1.0, 0.0, 0.0, float(WIN), S.TH_HIGH, cur_mp=sc.slot_owner())
    m.close()
    n_o, mp_o = O.search_by_projection_kf(O.OracleFrame(sc.kps, sc.desc, W, H), valid, world, md, sc.qdesc, sc.qangle, T_ID,
                                          1.0, 1.0, 0.0, 0.0, float(WIN), S.TH_HIGH, check_orientation=ori, cur_mp=sc.slot_owner())
    assert n == n_o and np.array_equal(mp, mp_o)


@pytest.mark.parametrize("name", ["chains-rule1", "tails-rule1", "ties-rule1"])
def test_window_search_and_f1f2(gpu_required, name):
    """Rule 1 through WindowSearch (F1 features at the window centres, window 6; no occupied slots, so the queries whose
    list holds an occupied slot are left out) and SearchByProjection(F1, F2, 6) (occupied slots as F2's map points)."""
    sc = scene(name)
    f1k = _last_frame(sc)
    m = fe.ORBmatcher(sc.nnratio, True)
    f1, f2 = M.FrameView(f1k, sc.qdesc, W, H), M.FrameView(sc.kps, sc.desc, W, H)
    o1, o2 = O.OracleFrame(f1k, sc.qdesc, W, H), O.OracleFrame(sc.kps, sc.desc, W, H)
    has, _ = S.window_search_view(sc)
    n, m21 = M.window_search(m, f1, f2, has, WIN)
    n_o, m21_o = O.window_search(o1, o2, has, WIN, nnratio=sc.nnratio, check_orientation=True)
    assert n == n_o > 0 and np.array_equal(m21, m21_o)
    valid = np.ones(sc.nq, np.uint8)
    n, mp = M.search_by_projection_f1f2(m, f1, f2, valid, _world(sc), T_ID, 1.0, 1.0, 0.0, 0.0, WIN, f2_mp=sc.slot_owner())
    n_o, mp_o = O.search_by_projection_f1f2(o1, o2, valid, _world(sc), T_ID, 1.0, 1.0, 0.0, 0.0, WIN, nnratio=sc.nnratio,
                                            f2_mp=sc.slot_owner())
    m.close()
    assert n == n_o == S.sequential(sc)[0] and np.array_equal(mp, mp_o)


@pytest.mark.parametrize("name", ["chains-rule2", "tails-rule2"])
def test_search_local_points(gpu_required, name):
    """Rule 2 through SearchByProjection(Frame, vector<MapPoint*>, th = 1.25): predicted level 1, view cosine 0 (radius 4),
    so the window is 4 * 1.25 * 1.2 px over octaves 0..1."""
    sc = scene(name)
    npt = sc.nq
    iv, lv, vc = np.ones(npt, np.uint8), np.ones(npt, np.int32), np.zeros(npt, np.float32)
    xy = np.stack([sc.qu, sc.qv], 1).astype(np.float32)
    m = fe.ORBmatcher(sc.nnratio, False)
    n, mp = M.search_local_points(m, M.FrameView(sc.kps, sc.desc, W, H), iv, xy, lv, vc, sc.qdesc, 1.25, f_mp=sc.slot_owner())
    m.close()
    n_o, mp_o = O.search_local_points(O.OracleFrame(sc.kps, sc.desc, W, H), iv, xy, lv, vc, sc.qdesc, 1.25, nnratio=sc.nnratio,
                                      f_mp=sc.slot_owner())
    assert n == n_o == S.sequential(sc)[0] and np.array_equal(mp, mp_o)


@pytest.mark.parametrize("ori", [False, True])
def test_search_for_initialization(gpu_required, ori):
    """MODE 2: the prefetched-distance patch, the re-assignment chain with its stale histogram entries, lists of 32 and 40
    entries, TH_LOW 50 / 51 and the strict ratio test at equality; host and device forms, vnMatches12 and vbPrevMatched."""
    import torch
    sc = scene("init")
    f1k = _last_frame(sc)
    prev = np.stack([sc.qu, sc.qv], 1).astype(np.float32)
    m = fe.ORBmatcher(sc.nnratio, ori)
    n, m12, pv = M.search_for_initialization(m, M.FrameView(f1k, sc.qdesc, W, H), M.FrameView(sc.kps, sc.desc, W, H), prev, WIN)
    n_o, m12_o, pv_o = O.search_for_initialization(O.OracleFrame(f1k, sc.qdesc, W, H), O.OracleFrame(sc.kps, sc.desc, W, H), prev,
                                                   WIN, nnratio=sc.nnratio, check_orientation=ori)
    assert n == n_o and np.array_equal(m12, m12_o) and np.array_equal(pv, pv_o)
    cap = max(sc.n, sc.nq)
    kps = np.zeros((2, cap), fe.KP_DTYPE)
    desc = np.zeros((2, cap, 32), np.uint8)
    kps[0, :sc.nq], desc[0, :sc.nq], kps[1, :sc.n], desc[1, :sc.n] = f1k, sc.qdesc, sc.kps, sc.desc
    pr = np.zeros((1, cap, 2), np.float32)
    pr[0, :sc.nq] = prev
    dev = torch.device("cuda", 0)
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev)
    d_prev, d_m12 = t(pr), torch.full((1, cap), -7, dtype=torch.int32, device=dev)
    d_nm = torch.zeros(1, dtype=torch.int32, device=dev)
    d = [t(kps.view(np.uint8).reshape(2, cap, 28)), t(desc), t(np.array([sc.nq, sc.n], np.int32)), t(np.array([0], np.int32)),
         t(np.array([1], np.int32))]
    M.search_for_initialization_device(m, 1, d[0].data_ptr(), d[1].data_ptr(), d[2].data_ptr(), cap, d[3].data_ptr(), d[4].data_ptr(),
                                       d_prev.data_ptr(), W, H, WIN, d_m12.data_ptr(), d_nm.data_ptr())
    m.sync()
    m.close()
    assert int(d_nm.cpu()[0]) == n_o
    assert np.array_equal(d_m12.cpu().numpy()[0, :sc.nq], m12_o) and np.array_equal(d_prev.cpu().numpy()[0, :sc.nq], pv_o)


def test_chain_across_the_query_split(gpu_required):
    """A blocked rule-1 chain across the query split of orbfe_guided_search without the histogram: two launches, and the
    second one starts on slots the first one took."""
    sc = S.split_chain_scene()
    v, o = _views(sc)
    m = fe.ORBmatcher(sc.nnratio, False)
    args = (sc.qu, sc.qv, sc.qr, sc.qlo, sc.qhi, sc.qdesc, sc.qangle, 1)
    n0 = m.counters()[2]
    n, so = M.guided_search(m, v, *args, S.TH_HIGH, 0, slot_owner=sc.slot_owner())
    assert m.counters()[2] - n0 == 2
    m.close()
    n_o, so_o = O.guided_search(o, *args, sc.nnratio, S.TH_HIGH, 0, slot_owner=sc.slot_owner())
    assert n == n_o == len(sc.facts["chain"]) and np.array_equal(so, so_o)
