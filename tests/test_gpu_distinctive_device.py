"""GPU parity of the device-resident MapPoint::ComputeDistinctiveDescriptors (orbfe_distinctive_descriptors_device): map points
given as observation lists into the frame store, bit-exact against the oracle and the host entry orbfe_distinctive_descriptors
on the host-gathered descriptors, against the reference's own MapPoint.cc, and chained into orbfe_guided_search_device."""
import numpy as np
import pytest

import oracle as O
import orb_slam_b200 as fe
from oracle import ref as R
from orb_slam_b200 import bow as B
from orb_slam_b200 import matching as M
from orb_slam_b200.synth import noisy_copies, random_descriptors, shifted_frame, textured_frame

pytestmark = pytest.mark.gpu

SENTINEL = 0xA5


def _torch():
    import torch
    return torch, torch.device("cuda", 0)


def _csr(groups):
    ptr = np.concatenate([[0], np.cumsum([len(g) for g in groups])]).astype(np.int32)
    obs = np.concatenate([np.asarray(g, np.int32) for g in groups] + [np.zeros(0, np.int32)]).astype(np.int32)
    return ptr, obs


def _run_device(m, desc, counts, ptr, obs, nobs=None):
    """One call on a user stream; returns (best, mp_desc rows).  mp_desc is prefilled with SENTINEL."""
    torch, dev = _torch()
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev)
    F, cap = desc.shape[:2]
    ng = len(ptr) - 1
    d_desc, d_cnt, d_ptr, d_obs = t(desc), t(counts), t(ptr), t(obs if len(obs) else np.zeros(1, np.int32))
    d_best = torch.full((ng,), -9, dtype=torch.int32, device=dev)
    d_mp = torch.full((ng, 32), SENTINEL, dtype=torch.uint8, device=dev)
    s = torch.cuda.Stream(device=dev)
    torch.cuda.synchronize()
    B.distinctive_descriptors_device(m, ng, d_desc.data_ptr(), d_cnt.data_ptr(), F, cap, d_ptr.data_ptr(), d_obs.data_ptr(),
                                     len(obs) if nobs is None else nobs, d_best.data_ptr(), d_mp.data_ptr(), s.cuda_stream)
    s.synchronize()
    return d_best.cpu().numpy(), d_mp.cpu().numpy()


# ---------------------------------------------------------------------------------------------------------------------
# The seeded frame store
# ---------------------------------------------------------------------------------------------------------------------
SIZES = [0, 1, 2, 31, 32, 33, 64, 400, 1500]


def _store(seed, nframes=40, cap=2048, ngroups=3000, nperm=200):
    """nframes frames of varying counts (frame 3 empty); groups of the SIZES above plus mostly 2-10 observations with a
    tail up to 150, each on distinct slots, as noisy copies of one descriptor per group.  Every tenth group has an exact
    duplicate pair and a few are all one descriptor (median ties).  The last `nperm` groups repeat earlier groups that have
    a duplicate pair with their observations permuted.  Returns (desc, counts, groups, perm_of)."""
    rng = np.random.default_rng(seed)
    counts = rng.integers(800, cap + 1, nframes).astype(np.int32)
    counts[3] = 0
    desc = np.zeros((nframes, cap, 32), np.uint8)
    desc[:] = random_descriptors(nframes * cap, seed).reshape(nframes, cap, 32)
    flat = desc.reshape(-1, 32)
    slots = np.concatenate([f * cap + np.arange(counts[f]) for f in range(nframes)])
    slots = slots[rng.permutation(len(slots))].astype(np.int32)
    n_rest = ngroups - nperm - len(SIZES)
    sizes = np.where(rng.random(n_rest) < 0.95, rng.integers(2, 11, n_rest), rng.integers(11, 151, n_rest))
    sizes = np.concatenate([SIZES, sizes])
    rng.shuffle(sizes)
    groups, dup, at = [], [], 0
    for g, n in enumerate(sizes):
        sl = slots[at:at + n]
        at += n
        if n:
            flat[sl] = noisy_copies(np.repeat(random_descriptors(1, 7000 + g), n, axis=0), rng.uniform(0.02, 0.3), 9000 + g)
        if n >= 2 and g % 10 == 0:
            a, b = rng.choice(n, 2, replace=False)
            flat[sl[b]] = flat[sl[a]]
            dup.append(g)
        if 2 <= n <= 12 and g % 97 == 1:
            flat[sl] = flat[sl[0]]
            dup.append(g)
        groups.append(sl)
    assert at <= len(slots)
    perm_of = {}
    for g in rng.choice(dup, nperm, replace=len(dup) < nperm):
        perm_of[len(groups)] = int(g)
        groups.append(groups[g][rng.permutation(len(groups[g]))])
    return desc, counts, groups, perm_of


def _expected(desc, ptr, obs):
    gathered = desc.reshape(-1, 32)[obs]
    return gathered, O.distinctive_descriptors(gathered, ptr)


def test_distinctive_device_matches_oracle_and_host_entry(gpu_required):
    desc, counts, groups, perm_of = _store(5)
    ptr, obs = _csr(groups)
    flat = desc.reshape(-1, 32)
    m = fe.ORBmatcher(0.6, True)
    best, rows = _run_device(m, desc, counts, ptr, obs)
    m.sync()
    gathered, best_o = _expected(desc, ptr, obs)
    best_h = B.distinctive_descriptors(m, gathered, ptr)
    assert np.array_equal(best, best_o) and np.array_equal(best_h, best_o)
    sizes = np.diff(ptr)
    assert set(SIZES) <= set(sizes.tolist()) and len(groups) >= 3000
    for g in range(len(groups)):
        if sizes[g] == 0:
            assert best[g] == -1 and (rows[g] == SENTINEL).all(), g
        else:
            assert 0 <= best[g] < sizes[g] and np.array_equal(rows[g], flat[obs[ptr[g] + best[g]]]), g
    # the position follows the given order: a permuted group picks another slot of the same bytes when a tie moved first
    moved = sum(obs[ptr[p] + best[p]] != obs[ptr[g] + best[g]] for p, g in perm_of.items())
    assert moved > 10, moved
    m.close()


# ---------------------------------------------------------------------------------------------------------------------
# The reference's own MapPoint::ComputeDistinctiveDescriptors
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.skipif(not R.available("ref"), reason="oracle/_ref is not built")
def test_distinctive_device_against_the_reference(gpu_required):
    """Keyframes of the reference's map model and the same descriptors in a device frame store (keyframe k = frame k);
    each map point's observation list in the order of its std::map, as the caller builds it from GetObservations()."""
    import ctypes as C
    S = R.Scene("ref")
    L = S.L
    L.ref_mp_observation_order.argtypes = [C.c_int, C.c_void_p, C.c_void_p, C.c_int]
    rng = np.random.default_rng(8)
    nkf, nfeat, cap = 12, 80, 96
    base = random_descriptors(nfeat, 21)
    kps = np.zeros(nfeat, O.KP_DTYPE)
    kps["x"], kps["y"] = rng.uniform(20, 600, nfeat), rng.uniform(20, 440, nfeat)
    store = np.zeros((nkf, cap, 32), np.uint8)
    kfs = []
    for k in range(nkf):
        d = noisy_copies(base, 0.10, 300 + k)
        if k:   # exact copies of keyframe 0's descriptors: median ties decided by the observation order
            same = rng.random(nfeat) < 0.15
            d[same] = store[0, :nfeat][same]
        store[k, :nfeat] = d
        f = S.frame(kps, d, 640, 480, 500.0, 500.0, 320.0, 240.0)
        kfs.append(S.keyframe(f, np.eye(4, dtype=np.float32)[:3]))
        f.close()
    groups, want = [], []
    for i in range(nfeat):
        mp = S.map_point(np.array([0, 0, 4], np.float32), store[0, i], None, 1.0, 30.0, kfs[0])
        seen = [k for k in range(nkf) if rng.random() < 0.6] or [0]
        if i % 9 == 0:
            seen = list(range(nkf))
        for k in seen:
            S.observe(kfs[k], mp, i)
        want.append(S.compute_distinctive(mp))
        ok_, oi_ = np.zeros(nkf, np.int32), np.zeros(nkf, np.int32)
        n = L.ref_mp_observation_order(mp, ok_.ctypes.data, oi_.ctypes.data, nkf)
        groups.append(np.array([kfs.index(int(ok_[j])) * cap + int(oi_[j]) for j in range(n)], np.int32))
    ptr, obs = _csr(groups)
    counts = np.full(nkf, nfeat, np.int32)
    m = fe.ORBmatcher(0.6, True)
    best, rows = _run_device(m, store, counts, ptr, obs)
    m.sync()
    for i in range(nfeat):
        assert np.array_equal(rows[i], want[i]), i
    assert np.array_equal(best, _expected(store, ptr, obs)[1])
    m.close()


# ---------------------------------------------------------------------------------------------------------------------
# The whole chain on the device: extraction -> distinctive descriptors -> guided search
# ---------------------------------------------------------------------------------------------------------------------
def test_device_chain_extract_distinctive_guided_search(gpu_required):
    """orbfe_extract_batch_device on shifted frames, the map points' observation lists from the known image shifts, then
    orbfe_distinctive_descriptors_device, whose d_mp_desc is the d_qdesc of one orbfe_guided_search_device job that
    searches a frame the points were not observed in.  Only the observation arrays go from the host to the device on
    the way; the host knows the keypoints as a SLAM system's frames do (the host extraction, which the device one equals).
    The matches equal the same job run with the oracle's descriptors uploaded from the host."""
    torch, dev = _torch()
    W, H, NF, NL = 640, 480, 1000, 8
    base = textured_frame(W, H, seed=31)
    shifts = [(0, 0), (3, -2), (-4, 1), (6, 3), (-2, -5), (5, 4)]
    frames = np.stack([base] + [shifted_frame(base, dx, dy, seed=i) for i, (dx, dy) in enumerate(shifts) if i])
    Bn, T = len(frames), len(frames) - 1   # frames 0..T-1 observe the map points, frame T is searched
    ex = fe.ORBextractor(NF, 1.2, NL)
    hk, _, hc = ex.extract_batch(frames)
    groups, q = [], []
    for i in range(hc[0]):
        x0, y0, o0 = hk[0, i]["x"], hk[0, i]["y"], hk[0, i]["octave"]
        g = [i]
        for f in range(1, T):
            k = hk[f, :hc[f]]
            d2 = (k["x"] - x0 - shifts[f][0]) ** 2 + (k["y"] - y0 - shifts[f][1]) ** 2
            j = int(np.argmin(d2))
            if d2[j] < 0.25 and k[j]["octave"] == o0:
                g.append(f * NF + j)
        if len(g) >= 2:
            groups.append(g)
            q.append((x0 + shifts[T][0], y0 + shifts[T][1], 4.0 * 1.2 ** o0, hk[0, i]["angle"]))
    ptr, obs = _csr(groups)
    ng = len(groups)
    assert ng > 300 and np.diff(ptr).max() >= T, (ng, np.diff(ptr).max())
    q = np.array(q, np.float32)
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev)
    d_frames = torch.from_numpy(frames).to(dev)
    d_kps = torch.zeros((Bn, NF, 28), dtype=torch.uint8, device=dev)
    d_desc = torch.zeros((Bn, NF, 32), dtype=torch.uint8, device=dev)
    d_cnt = torch.zeros((Bn,), dtype=torch.int32, device=dev)
    d_ptr, d_obs = t(ptr), t(obs)
    d_best = torch.zeros(ng, dtype=torch.int32, device=dev)
    d_mp = torch.zeros((ng, 32), dtype=torch.uint8, device=dev)
    d_qu, d_qv, d_qr, d_qa = (t(q[:, c]) for c in range(4))
    d_qlo = d_qhi = torch.full((ng,), -1, dtype=torch.int32, device=dev)
    d_fi, d_qb, d_qc = t(np.array([T], np.int32)), t(np.array([0], np.int32)), t(np.array([ng], np.int32))
    m = fe.ORBmatcher(0.8, True)

    def guided(d_qdesc):
        so, nm = torch.full((1, NF), -1, dtype=torch.int32, device=dev), torch.zeros(1, dtype=torch.int32, device=dev)
        M.guided_search_device(m, 1, d_kps.data_ptr(), d_desc.data_ptr(), d_cnt.data_ptr(), NF, d_fi.data_ptr(), d_qu.data_ptr(),
                               d_qv.data_ptr(), d_qr.data_ptr(), d_qlo.data_ptr(), d_qhi.data_ptr(), d_qdesc.data_ptr(), d_qa.data_ptr(),
                               d_qb.data_ptr(), d_qc.data_ptr(), ng, W, H, 2, 0, so.data_ptr(), nm.data_ptr(), s.cuda_stream)
        return so, nm

    s = torch.cuda.Stream(device=dev)
    torch.cuda.synchronize()
    ex.extract_batch_device(d_frames.data_ptr(), W, H, W, W * H, Bn, d_kps.data_ptr(), d_desc.data_ptr(), d_cnt.data_ptr(), s.cuda_stream)
    B.distinctive_descriptors_device(m, ng, d_desc.data_ptr(), d_cnt.data_ptr(), Bn, NF, d_ptr.data_ptr(), d_obs.data_ptr(), len(obs),
                                     d_best.data_ptr(), d_mp.data_ptr(), s.cuda_stream)
    so_dev, nm_dev = guided(d_mp)
    s.synchronize()
    m.sync()
    kps, desc, counts = d_kps.cpu().numpy().view(fe.KP_DTYPE).reshape(Bn, NF), d_desc.cpu().numpy(), d_cnt.cpu().numpy()
    assert np.array_equal(counts, hc)
    for f in range(Bn):
        assert all(np.array_equal(kps[f, :hc[f]][k], hk[f, :hc[f]][k]) for k in ("x", "y", "octave")), f
    gathered, best_o = _expected(desc, ptr, obs)
    assert np.array_equal(d_best.cpu().numpy(), best_o)
    chosen = gathered[ptr[:-1] + best_o]
    assert np.array_equal(d_mp.cpu().numpy(), chosen)
    so_host, nm_host = guided(t(chosen))
    s.synchronize()
    m.sync()
    assert nm_dev.item() == nm_host.item() and np.array_equal(so_dev.cpu().numpy(), so_host.cpu().numpy())
    assert nm_dev.item() > 200, nm_dev.item()
    ex.close()
    m.close()


# ---------------------------------------------------------------------------------------------------------------------
# Malformed input is never followed
# ---------------------------------------------------------------------------------------------------------------------
def test_malformed_groups_fail_only_themselves(gpu_required):
    """A feature index >= the frame's count, a frame >= nframes, a negative slot, a decreasing group pointer, a negative
    one and a last pointer beyond nobs, in one launch with good groups: the bad groups give -1 and keep their rows, the
    good ones are exact, the sync reports ORBFE_ERR_ARG naming the call once."""
    desc, counts, groups, _ = _store(9, nframes=12, cap=1024, ngroups=400, nperm=0)
    F, cap = desc.shape[:2]
    groups = [g[:40] for g in groups]
    f = next(f for f in range(F) if 0 < counts[f] < cap)   # a frame with room beyond its count
    big = [i for i, g in enumerate(groups) if len(g) >= 3][::5]
    groups[big[0]] = np.concatenate([groups[big[0]][:2], [f * cap + counts[f]], groups[big[0]][2:]]).astype(np.int32)
    groups[big[1]] = np.concatenate([groups[big[1]], [F * cap + 5]]).astype(np.int32)
    groups[big[2]] = np.concatenate([[-cap], groups[big[2]]]).astype(np.int32)
    ptr, obs = _csr(groups)
    ng = len(groups)
    ptr[big[3] + 1] = ptr[big[3]] - 1   # group big[3] decreasing; group big[3] + 1 starts earlier but stays valid
    ptr[big[4] + 1] = -3                 # group big[4] decreasing, big[4] + 1 starts below 0
    ptr[ng] = len(obs) + 4               # the last group ends beyond nobs
    m = fe.ORBmatcher(0.6, True)
    best, rows = _run_device(m, desc, counts, ptr, obs)
    with pytest.raises(fe.OrbfeError) as e:
        m.sync()
    assert e.value.code == fe.ORBFE_ERR_ARG and "orbfe_distinctive_descriptors_device" in str(e.value)
    m.sync()   # the flag is cleared by the report
    flat = desc.reshape(-1, 32)
    bad = []
    for g in range(ng):
        b, e_ = int(ptr[g]), int(ptr[g + 1])
        o = obs[b:e_] if 0 <= b <= e_ <= len(obs) else None
        if o is None or ((o < 0) | (o // cap >= F)).any() or (o % cap >= counts[np.minimum(o // cap, F - 1)]).any():
            bad.append(g)
            assert best[g] == -1 and (rows[g] == SENTINEL).all(), g
            continue
        if len(o) == 0:
            assert best[g] == -1 and (rows[g] == SENTINEL).all(), g
            continue
        bo = O.distinctive_descriptors(flat[o], np.array([0, len(o)], np.int32))[0]
        assert best[g] == bo and np.array_equal(rows[g], flat[o[bo]]), g
    assert sorted(bad) == sorted([big[0], big[1], big[2], big[3], big[4], big[4] + 1, ng - 1]), bad
    m.close()
