"""GPU parity of the matchers (the fused windowed kernel, the BoW kernels and the Hamming kernels, all through the C-ABI of
liborbfe.so) against the oracle's restatement of ORBmatcher.cc / Frame.cc."""
import numpy as np
import pytest

import oracle as O
import orb_slam_b200 as fe
from orb_slam_b200 import matching as M
from orb_slam_b200.synth import textured_frame, shifted_frame

pytestmark = pytest.mark.gpu

W, H = 640, 480
FX = FY = 500.0
CX, CY, DEPTH = W / 2.0, H / 2.0, 4.0


def _features(n_frames=3):
    ex = fe.ORBextractor(1000, 1.2, 8)
    base = textured_frame(W, H, seed=21)
    frames, shifts = [base], [(0, 0)]
    rng = np.random.default_rng(1)
    for i in range(1, n_frames):
        dx, dy = int(rng.integers(-5, 6)), int(rng.integers(-4, 5))
        frames.append(shifted_frame(frames[-1], dx, dy, seed=i))
        shifts.append((dx, dy))
    feats = [ex(f) for f in frames]
    ex.close()
    return feats, shifts


def _tcw(dx, dy):
    T = np.zeros((3, 4), np.float32)
    T[0, 0] = T[1, 1] = T[2, 2] = 1
    T[0, 3], T[1, 3] = dx * DEPTH / FX, dy * DEPTH / FY
    return T


def _world(k):
    w = np.empty((len(k), 3), np.float32)
    w[:, 0] = (k["x"] - np.float32(CX)) / np.float32(FX) * np.float32(DEPTH)
    w[:, 1] = (k["y"] - np.float32(CY)) / np.float32(FY) * np.float32(DEPTH)
    w[:, 2] = DEPTH
    return w


def test_search_by_projection_pairs(gpu_required):
    feats, shifts = _features(4)
    m = fe.ORBmatcher(0.9, True)
    rng = np.random.default_rng(3)
    curs, lasts, has, outl, world, T, pre = [], [], [], [], [], [], []
    for i in range(1, 4):
        kc, dc = feats[i]
        kl, dl = feats[i - 1]
        curs.append(M.FrameView(kc, dc, W, H))
        lasts.append(M.FrameView(kl, dl, W, H))
        has.append((rng.random(len(kl)) < 0.9).astype(np.uint8))
        outl.append((rng.random(len(kl)) < 0.05).astype(np.uint8))
        world.append(_world(kl))
        T.append(_tcw(*shifts[i]))
        occ = np.full(len(kc), -1, np.int32)
        occ[rng.random(len(kc)) < 0.03] = 5  # a few already-occupied slots
        pre.append(occ)
    nm, mp = M.search_by_projection_frames(m, curs, lasts, has, outl, world, T, FX, FY, CX, CY, 15.0, cur_mp=pre)
    total = 0
    for j in range(3):
        fc = O.OracleFrame(curs[j].kps, curs[j].desc, W, H)
        fl = O.OracleFrame(lasts[j].kps, lasts[j].desc, W, H)
        n_o, mp_o = O.search_by_projection_ff(fc, fl, has[j], outl[j], world[j], T[j], FX, FY, CX, CY, 15.0, True, cur_mp=pre[j])
        assert nm[j] == n_o
        assert np.array_equal(mp[j], mp_o)
        total += n_o
    assert total > 300  # the synthetic stream really has true matches
    m.close()


def test_window_search_and_initialization(gpu_required):
    feats, shifts = _features(2)
    (k1, d1), (k2, d2) = feats
    f1, f2 = M.FrameView(k1, d1, W, H), M.FrameView(k2, d2, W, H)
    o1, o2 = O.OracleFrame(k1, d1, W, H), O.OracleFrame(k2, d2, W, H)
    has = (np.random.default_rng(0).random(len(k1)) < 0.8).astype(np.uint8)
    for nnratio, ori, win, lo, hi in [(0.9, True, 50, -1, 2 ** 31 - 1), (0.6, False, 100, 2, 5), (0.9, True, 200, -1, 2 ** 31 - 1)]:
        m = fe.ORBmatcher(nnratio, ori)
        n, m21 = M.window_search(m, f1, f2, has, win, lo, hi)
        n_o, m21_o = O.window_search(o1, o2, has, win, lo, hi, nnratio=nnratio, check_orientation=ori)
        assert n == n_o and np.array_equal(m21, m21_o)
        m.close()
    m = fe.ORBmatcher(0.9, True)
    prev = np.stack([k1["x"], k1["y"]], axis=1).astype(np.float32)
    n, m12, prev_out = M.search_for_initialization(m, f1, f2, prev, 100)
    n_o, m12_o, prev_o = O.search_for_initialization(o1, o2, prev, 100, nnratio=0.9, check_orientation=True)
    assert n == n_o and np.array_equal(m12, m12_o) and np.array_equal(prev_out, prev_o)
    assert n > 20
    # second round with the updated prev-matched positions (Tracking::Initialize calls it repeatedly)
    n2, m12b, _ = M.search_for_initialization(m, f1, f2, prev_out, 100)
    n2_o, m12b_o, _ = O.search_for_initialization(o1, o2, prev_o, 100, nnratio=0.9, check_orientation=True)
    assert n2 == n2_o and np.array_equal(m12b, m12b_o)
    m.close()


def test_device_resident_search_by_projection(gpu_required):
    """The fused device kernel (grid + candidates + distances + greedy + rotation filter) vs the oracle."""
    import torch
    feats, shifts = _features(5)
    cap = 1000
    nfr = len(feats)
    kps_all = np.zeros((nfr, cap), fe.KP_DTYPE)
    desc_all = np.zeros((nfr, cap, 32), np.uint8)
    counts = np.zeros(nfr, np.int32)
    world = np.zeros((nfr, cap, 3), np.float32)
    flags = np.zeros((nfr, cap), np.uint8)
    rng = np.random.default_rng(11)
    for f, (k, d) in enumerate(feats):
        n = len(k) - 37 * f  # different counts per frame
        counts[f] = n
        kps_all[f, :n], desc_all[f, :n] = k[:n], d[:n]
        world[f, :n] = _world(k[:n])
        flags[f, :n] = (rng.random(n) < 0.92)
    pairs = [(1, 0), (2, 1), (3, 2), (4, 3), (4, 0), (2, 2)]
    npairs = len(pairs)
    T = np.stack([_tcw(*shifts[c]) if c == l + 1 else _tcw(0, 0) for c, l in pairs]).astype(np.float32)
    pre = np.full((npairs, cap), -1, np.int32)
    pre[rng.random((npairs, cap)) < 0.02] = 7
    dev = torch.device("cuda", 0)
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev)
    d_kps, d_desc, d_cnt = t(kps_all.view(np.uint8).reshape(nfr, cap, 28)), t(desc_all), t(counts)
    d_world, d_flags, d_T = t(world), t(flags), t(T.reshape(npairs, 12))
    d_cur = t(np.array([p[0] for p in pairs], np.int32))
    d_last = t(np.array([p[1] for p in pairs], np.int32))
    d_mp, d_nm = t(pre), torch.zeros(npairs, dtype=torch.int32, device=dev)
    torch.cuda.synchronize()
    m = fe.ORBmatcher(0.9, True)
    M.search_by_projection_device(m, npairs, d_kps.data_ptr(), d_desc.data_ptr(), d_cnt.data_ptr(), cap, d_cur.data_ptr(),
                                  d_last.data_ptr(), d_world.data_ptr(), d_flags.data_ptr(), d_T.data_ptr(), W, H, 1.2, 8,
                                  FX, FY, CX, CY, 15.0, d_mp.data_ptr(), d_nm.data_ptr())
    m.sync()
    mp, nm = d_mp.cpu().numpy(), d_nm.cpu().numpy()
    tot = 0
    for j, (c, l) in enumerate(pairs):
        nc, nl = counts[c], counts[l]
        fc = O.OracleFrame(kps_all[c, :nc], desc_all[c, :nc], W, H)
        fl = O.OracleFrame(kps_all[l, :nl], desc_all[l, :nl], W, H)
        n_o, mp_o = O.search_by_projection_ff(fc, fl, flags[l, :nl], np.zeros(nl, np.uint8), world[l, :nl], T[j], FX, FY, CX, CY,
                                              15.0, True, cur_mp=pre[j, :nc])
        assert nm[j] == n_o, (j, nm[j], n_o)
        assert np.array_equal(mp[j, :nc], mp_o), j
        tot += n_o
    assert tot > 1000
    # without the orientation check
    m2 = fe.ORBmatcher(0.9, False)
    d_mp2 = t(pre)
    M.search_by_projection_device(m2, npairs, d_kps.data_ptr(), d_desc.data_ptr(), d_cnt.data_ptr(), cap, d_cur.data_ptr(),
                                  d_last.data_ptr(), d_world.data_ptr(), d_flags.data_ptr(), d_T.data_ptr(), W, H, 1.2, 8,
                                  FX, FY, CX, CY, 15.0, d_mp2.data_ptr(), d_nm.data_ptr())
    m2.sync()
    mp2, nm2 = d_mp2.cpu().numpy(), d_nm.cpu().numpy()
    for j, (c, l) in enumerate(pairs):
        nc, nl = counts[c], counts[l]
        fc = O.OracleFrame(kps_all[c, :nc], desc_all[c, :nc], W, H)
        fl = O.OracleFrame(kps_all[l, :nl], desc_all[l, :nl], W, H)
        n_o, mp_o = O.search_by_projection_ff(fc, fl, flags[l, :nl], np.zeros(nl, np.uint8), world[l, :nl], T[j], FX, FY, CX, CY,
                                              15.0, False, cur_mp=pre[j, :nc])
        assert nm2[j] == n_o and np.array_equal(mp2[j, :nc], mp_o)
    m.close()
    m2.close()


def test_local_points_reloc_and_f1f2_projection(gpu_required):
    """M3 (local-map points), M4 (Frame vs KeyFrame, relocalisation) and M6 (F1->F2 projection window): array-level
    C-ABI against the oracle's restatement."""
    feats, shifts = _features(2)
    (k1, d1), (k2, d2) = feats
    n1 = len(k1)
    rng = np.random.default_rng(5)
    f2v, o2 = M.FrameView(k2, d2, W, H), O.OracleFrame(k2, d2, W, H)
    f1v, o1 = M.FrameView(k1, d1, W, H), O.OracleFrame(k1, d1, W, H)
    dx, dy = shifts[1]
    occupied = np.full(len(k2), -1, np.int32)
    occupied[rng.random(len(k2)) < 0.03] = 3

    # ---- M3: map points with cached projections (Frame::isInFrustum fills them) ----
    in_view = (rng.random(n1) < 0.9).astype(np.uint8)
    proj = np.stack([k1["x"] + np.float32(dx) + rng.normal(0, 1.0, n1).astype(np.float32),
                     k1["y"] + np.float32(dy) + rng.normal(0, 1.0, n1).astype(np.float32)], axis=1).astype(np.float32)
    level = k1["octave"].astype(np.int32)
    view_cos = np.where(rng.random(n1) < 0.5, 0.9995, 0.95).astype(np.float32)
    for th, nnr in ((1.0, 0.8), (3.0, 0.8), (5.0, 0.6)):
        m = fe.ORBmatcher(nnr, True)
        n, mp = M.search_local_points(m, f2v, in_view, proj, level, view_cos, d1, th, f_mp=occupied)
        n_o, mp_o = O.search_local_points(o2, in_view, proj, level, view_cos, d1, th, nnratio=nnr, f_mp=occupied)
        assert n == n_o and np.array_equal(mp, mp_o)
        m.close()
    assert n > 200

    # ---- M4: keyframe map points projected with the current pose, predicted level from the distance ----
    world = _world(k1)
    min_dist = (DEPTH / np.float32(1.2) ** k1["octave"].astype(np.float32) * rng.uniform(0.8, 1.1, n1)).astype(np.float32)
    valid = (rng.random(n1) < 0.85).astype(np.uint8)
    T = _tcw(dx, dy)
    T[2, 3] = 0.3  # a little forward motion so that predicted levels vary
    for th, od, ori in ((10.0, 100, True), (3.0, 64, True), (10.0, 100, False)):
        m = fe.ORBmatcher(0.9, ori)
        n, mp = M.search_by_projection_kf(m, f2v, valid, world, min_dist, d1, k1["angle"], T, FX, FY, CX, CY, th, od, cur_mp=occupied)
        n_o, mp_o = O.search_by_projection_kf(o2, valid, world, min_dist, d1, k1["angle"], T, FX, FY, CX, CY, th, od, ori, cur_mp=occupied)
        assert n == n_o and np.array_equal(mp, mp_o)
        m.close()

    # ---- M6: F1 map points projected into F2 with F2's pose, same-octave window ----
    T2 = _tcw(dx, dy)
    for win, nnr in ((15, 0.9), (50, 0.7)):
        m = fe.ORBmatcher(nnr, True)
        n, mp = M.search_by_projection_f1f2(m, f1v, f2v, valid, world, T2, FX, FY, CX, CY, win, f2_mp=occupied)
        n_o, mp_o = O.search_by_projection_f1f2(o1, o2, valid, world, T2, FX, FY, CX, CY, win, nnratio=nnr, f2_mp=occupied)
        assert n == n_o and np.array_equal(mp, mp_o)
        m.close()
    assert n > 100


def test_search_by_bow_both_overloads(gpu_required):
    """M9: brute force inside equal vocabulary nodes (FeatureVectors as CSR), both overloads, against the oracle."""
    rng = np.random.default_rng(21)
    n1, n2 = 1500, 1400
    d1 = M.np.zeros((0, 32), np.uint8)
    from orb_slam_b200.synth import random_descriptors, noisy_copies
    d1 = random_descriptors(n1, 5)
    perm = rng.permutation(n1)[:n2]
    d2 = noisy_copies(d1[perm], 0.05, 6)
    a1 = rng.uniform(0, 360, n1).astype(np.float32)
    a2 = ((a1[perm] + rng.normal(7, 4, n2)) % 360).astype(np.float32)
    # vocabulary node of a feature: a coarse function of a few descriptor bits (noisy copies mostly land in the same node)
    node1 = (d1[:, 0].astype(np.int32) >> 3) * 3 + 11
    node2 = (d2[:, 0].astype(np.int32) >> 3) * 3 + 11
    node2[rng.random(n2) < 0.05] = 9999  # a node that only one side has
    fv1, fv2 = M.feature_vector(node1), M.feature_vector(node2)
    valid1 = (rng.random(n1) < 0.8).astype(np.uint8)
    valid2 = (rng.random(n2) < 0.9).astype(np.uint8)
    for variant in (0, 1):
        for nnr, ori in ((0.75, True), (0.6, False)):
            m = fe.ORBmatcher(nnr, ori)
            n, out = M.search_by_bow(m, variant, d1, valid1, a1, fv1, d2, valid2, a2, fv2)
            n_o, out_o = O.search_by_bow(variant, d1, valid1, a1, fv1, d2, valid2, a2, fv2, nnratio=nnr, check_orientation=ori)
            assert n == n_o and np.array_equal(out, out_o), (variant, nnr, ori)
            assert n > 300
            m.close()


def test_guided_search_all_rules(gpu_required):
    """The exported guided-search skeleton (used by the KeyFrame-level facade methods) against the oracle, for every
    accept rule / histogram mode, with and without octave filters (KeyFrame::GetFeaturesInArea has none)."""
    feats, shifts = _features(2)
    (k1, d1), (k2, d2) = feats
    rng = np.random.default_rng(8)
    f2v, o2 = M.FrameView(k2, d2, W, H), O.OracleFrame(k2, d2, W, H)
    dx, dy = shifts[1]
    nq = len(k1)
    qu = (k1["x"] + np.float32(dx) + rng.normal(0, 1.5, nq)).astype(np.float32)
    qv = (k1["y"] + np.float32(dy) + rng.normal(0, 1.5, nq)).astype(np.float32)
    qr = (np.float32(6.0) * np.float32(1.2) ** k1["octave"]).astype(np.float32)
    occ = np.full(len(k2), -1, np.int32)
    occ[rng.random(len(k2)) < 0.02] = 1
    for rule, th, hist, filt in ((0, 50, 0, False), (0, 100, 1, True), (1, 0, 2, True), (2, 0, 0, True), (0, 64, 1, False)):
        lo = (k1["octave"] - 1).astype(np.int32) if filt else np.full(nq, -1, np.int32)
        hi = (k1["octave"]).astype(np.int32) if filt else np.full(nq, -1, np.int32)
        m = fe.ORBmatcher(0.8, True)
        n, so = M.guided_search(m, f2v, qu, qv, qr, lo, hi, d1, k1["angle"], rule, th, hist, slot_owner=occ)
        n_o, so_o = O.guided_search(o2, qu, qv, qr, lo, hi, d1, k1["angle"], rule, 0.8, th, hist, slot_owner=occ)
        assert n == n_o and np.array_equal(so, so_o), (rule, th, hist, filt)
        assert n > 100
        # the slot-free variant used by Fuse / SearchBySim3
        lo2 = (k1["octave"] - 1).astype(np.int32)
        hi2 = k1["octave"].astype(np.int32)
        bi = M.guided_best(m, f2v, qu, qv, qr, lo2, hi2, d1, 50 if rule == 0 else 100)
        bi_o = O.guided_best(o2, qu, qv, qr, lo2, hi2, d1, 50 if rule == 0 else 100)
        assert np.array_equal(bi, bi_o) and (bi >= 0).sum() > 100
        m.close()


def test_device_resident_guided_search(gpu_required):
    """orbfe_guided_search_device: several jobs with different frames / query counts / occupied slots in one launch,
    every accept rule, against the oracle."""
    import torch
    feats, shifts = _features(4)
    cap = 1000
    nfr = len(feats)
    kps_all = np.zeros((nfr, cap), fe.KP_DTYPE)
    desc_all = np.zeros((nfr, cap, 32), np.uint8)
    counts = np.zeros(nfr, np.int32)
    for f, (k, d) in enumerate(feats):
        n = len(k) - 23 * f
        counts[f] = n
        kps_all[f, :n], desc_all[f, :n] = k[:n], d[:n]
    rng = np.random.default_rng(17)
    jobs = [(1, 0), (2, 1), (3, 2), (0, 3), (2, 2)]  # (searched frame, frame the queries come from)
    qu, qv, qr, qlo, qhi, qd, qa, qbase, qcnt = [], [], [], [], [], [], [], [], []
    for tgt, src in jobs:
        k, d = feats[src]
        keep = rng.random(len(k)) < 0.8
        k, d = k[keep], d[keep]
        dx = sum(s[0] for s in shifts[src + 1:tgt + 1]) if tgt > src else -sum(s[0] for s in shifts[tgt + 1:src + 1])
        dy = sum(s[1] for s in shifts[src + 1:tgt + 1]) if tgt > src else -sum(s[1] for s in shifts[tgt + 1:src + 1])
        qbase.append(sum(qcnt))
        qcnt.append(len(k))
        qu.append(k["x"] + np.float32(dx) + rng.normal(0, 1.0, len(k)).astype(np.float32))
        qv.append(k["y"] + np.float32(dy) + rng.normal(0, 1.0, len(k)).astype(np.float32))
        qr.append((np.float32(7.0) * np.float32(1.2) ** k["octave"]).astype(np.float32))
        nofilt = rng.random(len(k)) < 0.2
        qlo.append(np.where(nofilt, -1, k["octave"] - 1).astype(np.int32))
        qhi.append(np.where(nofilt, -1, k["octave"] + (rng.random(len(k)) < 0.5)).astype(np.int32))
        qd.append(d)
        qa.append(k["angle"])
    cat = lambda xs, t: np.ascontiguousarray(np.concatenate(xs).astype(t))
    QU, QV, QR, QA = cat(qu, np.float32), cat(qv, np.float32), cat(qr, np.float32), cat(qa, np.float32)
    QLO, QHI, QD = cat(qlo, np.int32), cat(qhi, np.int32), np.ascontiguousarray(np.concatenate(qd))
    njobs, qcap = len(jobs), max(qcnt)
    pre = np.full((njobs, cap), -1, np.int32)
    pre[rng.random((njobs, cap)) < 0.03] = 4
    dev = torch.device("cuda", 0)
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev)
    d_kps, d_desc, d_cnt = t(kps_all.view(np.uint8).reshape(nfr, cap, 28)), t(desc_all), t(counts)
    d_fi = t(np.array([j[0] for j in jobs], np.int32))
    d_q = [t(x) for x in (QU, QV, QR, QLO, QHI, QD, QA)]
    d_qb, d_qc = t(np.array(qbase, np.int32)), t(np.array(qcnt, np.int32))
    total = 0
    for rule, th, ori in ((0, 60, True), (0, 100, False), (1, 0, False), (2, 0, False), (1, 0, True)):
        m = fe.ORBmatcher(0.8, ori)
        d_so, d_nm = t(pre), torch.zeros(njobs, dtype=torch.int32, device=dev)
        torch.cuda.synchronize()
        M.guided_search_device(m, njobs, d_kps.data_ptr(), d_desc.data_ptr(), d_cnt.data_ptr(), cap, d_fi.data_ptr(),
                               *[x.data_ptr() for x in d_q], d_qb.data_ptr(), d_qc.data_ptr(), qcap, W, H, rule, th,
                               d_so.data_ptr(), d_nm.data_ptr())
        m.sync()
        so, nm = d_so.cpu().numpy(), d_nm.cpu().numpy()
        for j, (tgt, src) in enumerate(jobs):
            nc = counts[tgt]
            fr = O.OracleFrame(kps_all[tgt, :nc], desc_all[tgt, :nc], W, H)
            sl = slice(qbase[j], qbase[j] + qcnt[j])
            n_o, so_o = O.guided_search(fr, QU[sl], QV[sl], QR[sl], QLO[sl], QHI[sl], QD[sl], QA[sl], rule, 0.8, th,
                                        1 if ori else 0, slot_owner=pre[j, :nc])
            assert nm[j] == n_o, (rule, j, nm[j], n_o)
            assert np.array_equal(so[j, :nc], so_o), (rule, j)
            total += n_o
        m.close()
    assert total > 3000


def test_search_for_triangulation(gpu_required):
    """M10: BoW-node brute force + epipolar constraint between two keyframes (pure horizontal translation => the
    fundamental matrix of a rectified pair), against the oracle."""
    feats, shifts = _features(2)
    (k1, d1), (k2, d2) = feats
    rng = np.random.default_rng(31)
    has1 = (rng.random(len(k1)) < 0.4).astype(np.uint8)
    has2 = (rng.random(len(k2)) < 0.4).astype(np.uint8)
    node1 = (d1[:, 3].astype(np.int32) >> 4) * 7 + 2
    node2 = (d2[:, 3].astype(np.int32) >> 4) * 7 + 2
    fv1, fv2 = M.feature_vector(node1), M.feature_vector(node2)
    # x2' F12-style constraint used by the reference: l = x1' F12; a sideways-moving camera gives epipolar lines y = const
    F12 = np.array([[0, 0, 0], [0, 0, -1], [0, 1, float(-shifts[1][1])]], np.float32)
    sigma2 = (np.float32(1.2) ** np.arange(8, dtype=np.float32)) ** 2
    for ori in (True, False):
        m = fe.ORBmatcher(0.6, ori)
        n, m12 = M.search_for_triangulation(m, k1, d1, has1, fv1, k2, d2, has2, fv2, F12, sigma2)
        n_o, m12_o = O.search_for_triangulation(k1, d1, has1, fv1, k2, d2, has2, fv2, F12, sigma2, check_orientation=ori)
        assert n == n_o and np.array_equal(m12, m12_o)
        assert n > 20
        m.close()


def test_undistort_keypoints_and_image_bounds(gpu_required):
    """N1: Frame::UndistortKeyPoints / ComputeImageBounds on the device vs python-cv2 golden vectors and the oracle,
    bit-exact; host-array form, device in-place form, and the k1 == 0 shortcut."""
    import os
    import torch
    g = np.load(os.path.join(os.path.dirname(__file__), "golden", "opencv_undistort.npz"))
    K = g["K"]
    fx, fy, cx, cy = float(K[0, 0]), float(K[1, 1]), float(K[0, 2]), float(K[1, 2])
    n = len(g["pts"])
    kps = np.zeros(n, fe.KP_DTYPE)
    kps["x"], kps["y"] = g["pts"][:, 0], g["pts"][:, 1]
    kps["size"], kps["angle"], kps["response"], kps["octave"], kps["class_id"] = 31.0, 12.5, 40.0, np.arange(n) % 8, -1
    m = fe.ORBmatcher(0.9, True)
    for i, D in enumerate(g["coeffs"]):
        out = M.undistort_keypoints(m, kps, fx, fy, cx, cy, D)
        assert np.array_equal(out["x"].view(np.uint32), g["out_%d" % i][:, 0].view(np.uint32))
        assert np.array_equal(out["y"].view(np.uint32), g["out_%d" % i][:, 1].view(np.uint32))
        for f in ("size", "angle", "response", "octave", "class_id"):
            assert np.array_equal(out[f], kps[f])
        assert np.array_equal(out, O.undistort_keypoints(kps, fx, fy, cx, cy, D))
        assert np.array_equal(M.image_bounds(m, 640, 480, fx, fy, cx, cy, D), O.image_bounds(640, 480, fx, fy, cx, cy, D))
        # device form, in place
        d = torch.from_numpy(kps.view(np.uint8).reshape(n, 28).copy()).to("cuda:0")
        M.undistort_keypoints_device(m, d.data_ptr(), d.data_ptr(), n, fx, fy, cx, cy, D)
        m.sync()
        assert np.array_equal(d.cpu().numpy().reshape(-1).view(fe.KP_DTYPE), out)
    assert np.array_equal(M.undistort_keypoints(m, kps, fx, fy, cx, cy, [0, 0.2, 0.1, 0.1]), kps)
    assert list(M.image_bounds(m, 640, 480, fx, fy, cx, cy, [0, 0, 0, 0])) == [0, 0, 640, 480]
    m.close()
