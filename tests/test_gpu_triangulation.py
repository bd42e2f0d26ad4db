"""GPU parity of the device-resident SearchForTriangulation (orbfe_search_for_triangulation_device): batches of keyframe pairs,
bit-exact against the oracle's restatement of ORBmatcher.cc:852-1014 and against the host entry orbfe_search_for_triangulation
on the same arrays."""
import numpy as np
import pytest

import oracle as O
import orb_slam_b200 as fe
from orb_slam_b200 import bow as B
from orb_slam_b200 import matching as M
from orb_slam_b200.synth import noisy_copies, random_descriptors, random_vocabulary, shifted_frame, textured_frame

pytestmark = pytest.mark.gpu

NL, NKF = 8, 20
FX, FY, CX, CY = 520.0, 515.0, 320.0, 240.0
KMAT = np.array([[FX, 0, CX], [0, FY, CY], [0, 0, 1]], np.float32)


def _torch():
    import torch
    return torch, torch.device("cuda", 0)


def _sigma2(nlevels=NL, scale=1.2):
    """KeyFrame::GetSigma2: the squared per-level scale factors, accumulated in float as ORBextractor does."""
    sf = [np.float32(1.0)]
    for _ in range(1, nlevels):
        sf.append(np.float32(sf[-1] * np.float32(scale)))
    return np.array([s * s for s in sf], np.float32)


def _rotation(rng, deg):
    w = rng.normal(size=3)
    k = w / np.linalg.norm(w)
    th = np.deg2rad(deg)
    kx = np.array([[0, -k[2], k[1]], [k[2], 0, -k[0]], [-k[1], k[0], 0]])
    return (np.eye(3) + np.sin(th) * kx + (1 - np.cos(th)) * kx @ kx).astype(np.float32)


def _skew(t):
    return np.array([[0, -t[2], t[1]], [t[2], 0, -t[0]], [-t[1], t[0], 0]], np.float32)


def compute_f12(pose1, pose2):
    """LocalMapping::ComputeF12 (LocalMapping.cc:452-469) in float32: K1^-T [t12]x R12 K2^-1."""
    (R1w, t1w), (R2w, t2w) = pose1, pose2
    R12 = R1w @ R2w.T
    t12 = -R1w @ R2w.T @ t2w + t1w
    Kinv = np.linalg.inv(KMAT).astype(np.float32)
    return (Kinv.T @ _skew(t12) @ R12 @ Kinv).astype(np.float32)


def _epipolar_ok(kp1, kp2, F, sigma2):
    """CheckDistEpipolarLine (ORBmatcher.cc:136-153) with every float op rounded to float32."""
    f = np.float32
    x1, y1, x2, y2 = f(kp1["x"]), f(kp1["y"]), f(kp2["x"]), f(kp2["y"])
    a = x1 * F[0] + y1 * F[3] + F[6]
    b = x1 * F[1] + y1 * F[4] + F[7]
    c = x1 * F[2] + y1 * F[5] + F[8]
    num = a * x2 + b * y2 + c
    den = a * a + b * b
    if den == 0:
        return False
    return float(num * num / den) < 3.84 * float(sigma2[kp2["octave"]])


def _pack_fvs(fvs, cap):
    """Host FeatureVectors (ids, ptr, items) in the frame-slot layout of orbfe_feature_vector_device."""
    F = len(fvs)
    ids, items = np.zeros((F, cap), np.int32), np.zeros((F, cap), np.int32)
    ptr, n = np.zeros((F, cap + 1), np.int32), np.zeros(F, np.int32)
    for f, (i, p, t) in enumerate(fvs):
        ids[f, :len(i)], ptr[f, :len(p)], items[f, :len(t)], n[f] = i, p, t, len(i)
    return ids, ptr, items, n


def _unpack_fv(ids, ptr, items, n, f):
    k = int(n[f])
    return ids[f, :k], ptr[f, :k + 1], items[f, :ptr[f, k]]


# ---------------------------------------------------------------------------------------------------------------------
# The frame store: real epipolar geometry, controlled distances to the epipolar lines, duplicated descriptors
# ---------------------------------------------------------------------------------------------------------------------
E, U1, U2 = NKF + 1, NKF + 2, NKF + 3
DEGENERATE = 5   # the job (0, DEGENERATE) is also run with a fundamental matrix whose first two columns are zero


def _store(seed, cap=1600):
    """Frame 0 is the current keyframe, frames 1..NKF its covisible neighbours: views of one set of 3-D points from nearby
    poses.  Frame E has no features; frames U1 / U2 keep every feature in one node.  Points come in families of three with
    near-equal descriptors, so a side-1 feature often has several candidates within TH_LOW.  A neighbour's observation of a
    point that frame 0 also sees is moved off frame 0's epipolar line by 0..1.6 times the test's threshold, so that both
    outcomes of CheckDistEpipolarLine occur; some of them get a duplicate (same descriptor and octave, 0.5 px along the line,
    a higher index) for distance ties, and the nodes of odd frames list their items in descending order."""
    rng = np.random.default_rng(seed)
    sigma2 = _sigma2()
    npts = 1500
    fam = random_descriptors(npts // 3 + 1, seed)
    base = noisy_copies(np.repeat(fam, 3, axis=0)[:npts], 0.02, seed + 1)
    X = np.stack([rng.uniform(-4, 4, npts), rng.uniform(-3, 3, npts), rng.uniform(4, 12, npts)], 1).astype(np.float32)
    a0 = rng.uniform(0, 360, npts)
    F = NKF + 4
    poses = [(np.eye(3, dtype=np.float32), np.zeros(3, np.float32))]
    poses += [(_rotation(rng, 3.0), rng.normal(0, 0.3, 3).astype(np.float32)) for _ in range(1, F)]
    kps = np.zeros((F, cap), fe.KP_DTYPE)
    desc = np.zeros((F, cap, 32), np.uint8)
    counts = np.zeros(F, np.int32)
    nodes = [np.zeros(0, np.int32)] * F
    seen0 = np.full(npts, -1)
    dups = 0

    def observe(f, sel, ref=None):
        nonlocal dups
        R, t = poses[f]
        Xc = X[sel] @ R.T + t
        n = len(sel)
        k = np.zeros(n, fe.KP_DTYPE)
        k["x"] = FX * Xc[:, 0] / Xc[:, 2] + CX
        k["y"] = FY * Xc[:, 1] / Xc[:, 2] + CY
        k["octave"] = rng.integers(0, NL, n)
        ang = (a0[sel] + rng.normal(7, 4, n)) % 360
        wild = rng.random(n) < 0.1
        ang[wild] = rng.uniform(0, 360, wild.sum())
        k["angle"] = ang
        d = noisy_copies(base[sel], 0.04, 1000 * seed + f)
        extra_k, extra_d = [], []
        if ref is not None:   # move the observations of frame `ref`'s points off their epipolar lines
            F12 = compute_f12(poses[ref], poses[f]).reshape(-1)
            for j in range(n):
                i1 = seen0[sel[j]] if ref == 0 else -1
                if ref != 0:
                    i1 = ref_index[f].get(int(sel[j]), -1)
                if i1 < 0:
                    continue
                kp1 = kps[ref, i1]
                a = kp1["x"] * F12[0] + kp1["y"] * F12[3] + F12[6]
                b = kp1["x"] * F12[1] + kp1["y"] * F12[4] + F12[7]
                nrm = np.hypot(a, b)
                r = rng.uniform(0, 1.6) * np.sqrt(3.84 * sigma2[k["octave"][j]])
                k["x"][j] += r * a / nrm
                k["y"][j] += r * b / nrm
                if rng.random() < 0.08:
                    e = k[j].copy()
                    e["x"] += -0.5 * b / nrm
                    e["y"] += 0.5 * a / nrm
                    extra_k.append(e)
                    extra_d.append(d[j])
                    dups += 1
        if extra_k:
            k = np.concatenate([k, np.array(extra_k, fe.KP_DTYPE)])
            d = np.concatenate([d, np.array(extra_d, np.uint8)])
        n = len(k)
        kps[f, :n], desc[f, :n], counts[f] = k, d, n
        nodes[f] = (d[:, 0].astype(np.int32) >> 3) * 3 + 11
        return n

    sel0 = rng.permutation(npts)[:1300]
    observe(0, sel0)
    seen0[sel0] = np.arange(len(sel0))
    nodes[0][rng.random(len(sel0)) < 0.05] = 9999   # a node no neighbour has
    ref_index = {}
    for f in range(1, NKF + 1):
        observe(f, rng.permutation(npts)[:int(rng.integers(300, 1300))], ref=0)
    selu = rng.permutation(npts)[:1200]
    observe(U1, selu)
    ref_index[U2] = {int(p): i for i, p in enumerate(selu)}
    observe(U2, rng.permutation(npts)[:1100], ref=U1)
    nodes[U1][:] = 0
    nodes[U2][:] = 0
    assert counts.max() <= cap and dups > 50
    has_mp = (rng.random((F, cap)) < 0.25).astype(np.uint8)
    fvs = []
    for f in range(F):
        ids, ptr, items = M.feature_vector(nodes[f])
        if f % 2 == 1:   # descending items inside every node: list order is not index order
            items = np.concatenate([items[ptr[k]:ptr[k + 1]][::-1] for k in range(len(ids))] or [items])
        fvs.append((ids, ptr, items.astype(np.int32)))
    return kps, desc, counts, has_mp, fvs, poses, sigma2


J_DUP, J_U12, J_U21, J_DEG = NKF, NKF + 4, NKF + 5, NKF + 6   # job rows of the duplicate, one-node and degenerate jobs


def _jobs(poses):
    """Frame 0 against every neighbour (job j against frame j + 1), a duplicated job, empty sides, one node against one node,
    and the job (0, DEGENERATE) again with a fundamental matrix whose first two columns are zero (den == 0 for every line)."""
    jobs = [(0, f) for f in range(1, NKF + 1)] + [(0, 3), (0, E), (E, 0), (E, E), (U1, U2), (U2, U1), (0, DEGENERATE)]
    F12 = np.stack([compute_f12(poses[a], poses[b]).reshape(-1) for a, b in jobs]).astype(np.float32)
    F12[-1].reshape(3, 3)[:, :2] = 0
    return np.array(jobs, np.int32), F12


def _run_device(m, kps, desc, counts, has_mp, fv_slots, jobs, F12, sigma2):
    torch, dev = _torch()
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev)
    F, cap = desc.shape[:2]
    d_kps, d_desc, d_cnt, d_mp = t(kps.view(np.uint8).reshape(F, cap, 28)), t(desc), t(counts), t(has_mp)
    d_ids, d_ptr, d_items, d_n = (t(a) for a in fv_slots)
    d_i1, d_i2, d_F = t(jobs[:, 0]), t(jobs[:, 1]), t(F12)
    nj = len(jobs)
    d_out = torch.full((nj, cap), -9, dtype=torch.int32, device=dev)
    d_nm = torch.full((nj,), -9, dtype=torch.int32, device=dev)
    s = torch.cuda.Stream(device=dev)
    torch.cuda.synchronize()
    M.search_for_triangulation_device(m, nj, d_kps.data_ptr(), d_desc.data_ptr(), d_cnt.data_ptr(), cap, d_ids.data_ptr(),
                                      d_ptr.data_ptr(), d_items.data_ptr(), d_n.data_ptr(), d_mp.data_ptr(), d_i1.data_ptr(),
                                      d_i2.data_ptr(), d_F.data_ptr(), sigma2, d_out.data_ptr(), d_nm.data_ptr(), s.cuda_stream)
    s.synchronize()
    return d_out.cpu().numpy(), d_nm.cpu().numpy()


def _args(kps, desc, counts, has_mp, fvs, f1, f2):
    n1, n2 = counts[f1], counts[f2]
    return (kps[f1, :n1], desc[f1, :n1], has_mp[f1, :n1], fvs[f1], kps[f2, :n2], desc[f2, :n2], has_mp[f2, :n2], fvs[f2])


def _hamming(a, b):
    return int(np.unpackbits(np.bitwise_xor(a, b)).sum())


def _walk_witnesses(kps, desc, has_mp, fvs, f1, f2, F12, sigma2, m12):
    """From the matches of one job with orientation off: (beyond, tie) = the number of matches whose distance is above that
    of another candidate that was free and eligible (the walk went past the best), and of matches that won a distance tie
    by feature index against an eligible candidate that passes the epipolar test and comes first in the node's list.  A
    candidate no match took was free when every side-1 feature of its node was processed."""
    taken = set(int(x) for x in m12 if x >= 0)
    ids1, ptr1, it1 = fvs[f1]
    ids2, ptr2, it2 = fvs[f2]
    node2 = {int(i): it2[ptr2[k]:ptr2[k + 1]] for k, i in enumerate(ids2)}
    node1 = {int(x): int(ids1[k]) for k in range(len(ids1)) for x in it1[ptr1[k]:ptr1[k + 1]]}
    beyond = tie = 0
    for i1 in np.nonzero(m12 >= 0)[0]:
        i2 = int(m12[i1])
        cand = node2[node1[int(i1)]]
        d = _hamming(desc[f1, i1], desc[f2, i2])
        free = [int(c) for c in cand if not has_mp[f2, c] and int(c) not in taken]
        dists = [_hamming(desc[f1, i1], desc[f2, c]) for c in free]
        if any(dc < d for dc in dists if dc <= 50):
            beyond += 1
        pos = {int(c): p for p, c in enumerate(cand)}
        for c, dc in zip(free, dists):
            if dc == d and c > i2 and pos[c] < pos[i2] and _epipolar_ok(kps[f1, i1], kps[f2, c], F12, sigma2):
                tie += 1
                break
    return beyond, tie


# ---------------------------------------------------------------------------------------------------------------------
# 1. Batched jobs against the oracle and the host entry
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("seed", [3, 17, 40])
def test_search_for_triangulation_device_matches_oracle_and_host(gpu_required, seed):
    kps, desc, counts, has_mp, fvs, poses, sigma2 = _store(seed)
    slots = _pack_fvs(fvs, desc.shape[1])
    jobs, F12 = _jobs(poses)
    for ori in (False, True):
        m = fe.ORBmatcher(0.6, ori)
        out, nm = _run_device(m, kps, desc, counts, has_mp, slots, jobs, F12, sigma2)
        m.sync()
        beyond = tie = 0
        for j, (f1, f2) in enumerate(jobs):
            args = _args(kps, desc, counts, has_mp, fvs, f1, f2)
            n_o, m12_o = O.search_for_triangulation(*args, F12[j], sigma2, check_orientation=ori)
            n_h, m12_h = M.search_for_triangulation(m, *args, F12[j], sigma2)
            assert nm[j] == n_o == n_h, (seed, ori, j, f1, f2, nm[j], n_o, n_h)
            assert np.array_equal(out[j, :counts[f1]], m12_o) and np.array_equal(m12_h, m12_o), (seed, ori, j, f1, f2)
            if not ori and (j < NKF or j == J_U12):
                b, t = _walk_witnesses(kps, desc, has_mp, fvs, f1, f2, F12[j], sigma2, m12_o)
                beyond += b
                tie += t
        assert nm[:NKF].sum() > 2000, (seed, ori, nm[:NKF])
        assert nm[J_DUP] == nm[2] and nm[J_DEG] == 0 and nm[DEGENERATE - 1] > 0
        assert nm[J_U12] > 100 and nm[J_U21] > 100, (nm[J_U12], nm[J_U21])   # one node against one node, both ways
        if not ori:
            assert beyond > 20 and tie > 0, (seed, beyond, tie)
        else:
            assert nm[:NKF].sum() < n_total_off   # the rotation histogram removed matches
        n_total_off = int(nm[:NKF].sum())
        m.close()


# ---------------------------------------------------------------------------------------------------------------------
# 2. The whole chain on the device
# ---------------------------------------------------------------------------------------------------------------------
def test_device_chain_extract_undistort_fv_triangulation(gpu_required):
    """orbfe_extract_batch_device -> orbfe_undistort_keypoints_device (in place) -> orbfe_bow_descend_device ->
    orbfe_feature_vector_device -> orbfe_search_for_triangulation_device with no host copy in between; equal to the host
    orbfe_search_for_triangulation on the downloaded arrays and to the oracle."""
    torch, dev = _torch()
    W, H, NF, levelsup = 640, 480, 1000, 3
    base = textured_frame(W, H, seed=12)
    shifts = [(0, 0)] + [(3 * i - 7, 2 * i - 5) for i in range(1, 6)]
    frames = np.stack([base] + [shifted_frame(base, dx, dy, seed=i) for i, (dx, dy) in enumerate(shifts) if i])
    Bn = len(frames)
    dist = (0.02, 0.0, 0.0, 0.0)
    voc = random_vocabulary(10, 4, seed=6)
    v = B.Vocabulary(voc)
    ex = fe.ORBextractor(NF, 1.2, NL)
    sigma2 = _sigma2()
    rng = np.random.default_rng(4)
    d_frames = torch.from_numpy(frames).to(dev)
    d_mp = torch.from_numpy((rng.random((Bn, NF)) < 0.2).astype(np.uint8)).to(dev)
    d_kps = torch.zeros((Bn, NF, 28), dtype=torch.uint8, device=dev)
    d_desc = torch.zeros((Bn, NF, 32), dtype=torch.uint8, device=dev)
    d_cnt = torch.zeros((Bn,), dtype=torch.int32, device=dev)
    d_leaf = torch.zeros(Bn * NF, dtype=torch.int32, device=dev)
    d_node = torch.zeros(Bn * NF, dtype=torch.int32, device=dev)
    d_ids = torch.zeros((Bn, NF), dtype=torch.int32, device=dev)
    d_ptr = torch.zeros((Bn, NF + 1), dtype=torch.int32, device=dev)
    d_items = torch.zeros((Bn, NF), dtype=torch.int32, device=dev)
    d_n = torch.zeros((Bn,), dtype=torch.int32, device=dev)
    # job j: frame 0 (the new keyframe) against frame j + 1, plus one pair of neighbours; a sideways image shift (dx, dy)
    # puts the epipolar line of (x1, y1) at y2 = y1 + dy
    jobs = np.array([(0, f) for f in range(1, Bn)] + [(2, 4)], np.int32)
    F12 = np.zeros((len(jobs), 9), np.float32)
    for j, (f1, f2) in enumerate(jobs):
        F12[j, 5], F12[j, 7], F12[j, 8] = -1, 1, -(shifts[f2][1] - shifts[f1][1])
    d_i1, d_i2 = torch.from_numpy(jobs[:, 0].copy()).to(dev), torch.from_numpy(jobs[:, 1].copy()).to(dev)
    d_F = torch.from_numpy(F12).to(dev)
    d_out = torch.zeros((len(jobs), NF), dtype=torch.int32, device=dev)
    d_nm = torch.zeros(len(jobs), dtype=torch.int32, device=dev)
    m = fe.ORBmatcher(0.6, False)
    s = torch.cuda.Stream(device=dev)
    torch.cuda.synchronize()
    ex.extract_batch_device(d_frames.data_ptr(), W, H, W, W * H, Bn, d_kps.data_ptr(), d_desc.data_ptr(), d_cnt.data_ptr(), s.cuda_stream)
    M.undistort_keypoints_device(m, d_kps.data_ptr(), d_kps.data_ptr(), Bn * NF, FX, FY, CX, CY, dist, s.cuda_stream)
    v.descend_device(d_desc.data_ptr(), Bn * NF, levelsup, d_leaf.data_ptr(), d_node.data_ptr(), s.cuda_stream)
    B.feature_vector_device(v, Bn, d_leaf.data_ptr(), d_node.data_ptr(), d_cnt.data_ptr(), NF, d_ids.data_ptr(), d_ptr.data_ptr(),
                            d_items.data_ptr(), d_n.data_ptr(), s.cuda_stream)
    M.search_for_triangulation_device(m, len(jobs), d_kps.data_ptr(), d_desc.data_ptr(), d_cnt.data_ptr(), NF, d_ids.data_ptr(),
                                      d_ptr.data_ptr(), d_items.data_ptr(), d_n.data_ptr(), d_mp.data_ptr(), d_i1.data_ptr(),
                                      d_i2.data_ptr(), d_F.data_ptr(), sigma2, d_out.data_ptr(), d_nm.data_ptr(), s.cuda_stream)
    s.synchronize()
    m.sync()
    kps = d_kps.cpu().numpy().view(fe.KP_DTYPE).reshape(Bn, NF)
    desc, counts, has_mp = d_desc.cpu().numpy(), d_cnt.cpu().numpy(), d_mp.cpu().numpy()
    ids, ptr, items, n = (t.cpu().numpy() for t in (d_ids, d_ptr, d_items, d_n))
    fvs = [_unpack_fv(ids, ptr, items, n, f) for f in range(Bn)]
    out, nm = d_out.cpu().numpy(), d_nm.cpu().numpy()
    for f in range(Bn):
        assert all(np.array_equal(a, b) for a, b in zip(fvs[f], O.bow_transform(voc, desc[f, :counts[f]], levelsup)[1]))
    for j, (f1, f2) in enumerate(jobs):
        args = _args(kps, desc, counts, has_mp, fvs, f1, f2)
        n_h, m12_h = M.search_for_triangulation(m, *args, F12[j], sigma2)
        n_o, m12_o = O.search_for_triangulation(*args, F12[j], sigma2, check_orientation=False)
        assert nm[j] == n_h == n_o, j
        assert np.array_equal(out[j, :counts[f1]], m12_h) and np.array_equal(m12_h, m12_o), j
    assert nm.sum() > 200, nm
    ex.close(); v.close(); m.close()


# ---------------------------------------------------------------------------------------------------------------------
# 3. Malformed input is bounds-checked
# ---------------------------------------------------------------------------------------------------------------------
def test_malformed_frames_fail_only_their_jobs(gpu_required):
    """An out-of-range feature index (as side 2 and as side 1) and an out-of-range octave of a side-2 candidate make only
    their jobs -1; out-of-range octaves that are never read (a side-2 feature with a map point, side-1 features) do not."""
    kps, desc, counts, has_mp, fvs, poses, sigma2 = _store(5)
    bad_item, bad_octave, mp_octave = 7, 9, 11
    # one more frame: a copy of frame 12 whose octaves are all out of range, used only as side 1
    S1 = len(counts)
    kps, desc, has_mp = (np.concatenate([a, a[12:13]]) for a in (kps, desc, has_mp))
    counts, fvs, poses = np.append(counts, counts[12]).astype(np.int32), fvs + [fvs[12]], poses + [poses[12]]
    kps["octave"][S1, :counts[S1]] = 99
    cap = desc.shape[1]
    ids, ptr, items, n = _pack_fvs(fvs, cap)

    def node_row(f, nodes):
        return next(k for k, node in enumerate(fvs[f][0]) if int(node) in nodes)

    # one feature index of a node that frame 7 shares with frames 0 and 1 out of range
    k = node_row(bad_item, set(fvs[0][0].tolist()) & set(fvs[1][0].tolist()))
    items[bad_item, ptr[bad_item, k]] = counts[bad_item] + 5

    def feature_in_common_node(f, with_mp):
        fi, fp, ft = fvs[f]
        for k, node in enumerate(fi):
            if int(node) in set(fvs[0][0].tolist()):
                for i in ft[fp[k]:fp[k + 1]]:
                    if bool(has_mp[f, i]) == with_mp:
                        return int(i)
        raise AssertionError(f)

    kps["octave"][bad_octave, feature_in_common_node(bad_octave, False)] = NL   # read as a side-2 candidate: malformed
    kps["octave"][mp_octave, feature_in_common_node(mp_octave, True)] = -1      # has a map point: never read
    jobs, F12 = _jobs(poses)
    jobs = np.concatenate([jobs, [(bad_item, 1), (S1, 0)]]).astype(np.int32)
    F12 = np.concatenate([F12, [compute_f12(poses[bad_item], poses[1]).reshape(-1),
                                compute_f12(poses[S1], poses[0]).reshape(-1)]]).astype(np.float32)
    m = fe.ORBmatcher(0.6, True)
    out, nm = _run_device(m, kps, desc, counts, has_mp, (ids, ptr, items, n), jobs, F12, sigma2)
    with pytest.raises(fe.OrbfeError) as e:
        m.sync()
    assert e.value.code == fe.ORBFE_ERR_ARG and "orbfe_search_for_triangulation_device" in str(e.value)
    m.sync()   # the flag is cleared by the report
    checked = failed = 0
    for j, (f1, f2) in enumerate(jobs):
        if f1 == bad_item or f2 == bad_item or f2 == bad_octave:
            assert nm[j] == -1, (j, f1, f2)
            failed += 1
            continue
        n_o, m12_o = O.search_for_triangulation(*_args(kps, desc, counts, has_mp, fvs, f1, f2), F12[j], sigma2, check_orientation=True)
        assert nm[j] == n_o and np.array_equal(out[j, :counts[f1]], m12_o), (j, f1, f2)
        checked += 1
    assert failed == 3 and checked == len(jobs) - 3
    assert nm[mp_octave - 1] > 0 and nm[len(jobs) - 1] > 0
    m.close()
