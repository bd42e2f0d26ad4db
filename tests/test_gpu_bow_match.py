"""GPU parity of the device-resident SearchByBoW path: FeatureVectors built on the device (orbfe_feature_vector_device) and
SearchByBoW for batches of frame pairs (orbfe_search_by_bow_device), bit-exact against the host entry points and the
oracle's restatement of ORBmatcher.cc / DBoW2."""
import numpy as np
import pytest

import oracle as O
import orb_slam_b200 as fe
from orb_slam_b200 import bow as B
from orb_slam_b200 import matching as M
from orb_slam_b200.synth import noisy_copies, random_descriptors, random_vocabulary, shifted_frame, textured_frame

pytestmark = pytest.mark.gpu


def _torch():
    import torch
    return torch, torch.device("cuda", 0)


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


def _fv_equal(a, b):
    return all(np.array_equal(x, y) for x, y in zip(a, b))


# ---------------------------------------------------------------------------------------------------------------------
# 1. FeatureVector on the device
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("k,L,ragged,levelsup", [(10, 4, False, 2), (10, 4, False, 0), (10, 4, False, 4), (10, 4, False, 5), (7, 3, True, 1)])
def test_feature_vector_device_matches_host_and_oracle(gpu_required, k, L, ragged, levelsup):
    torch, dev = _torch()
    voc = random_vocabulary(k, L, seed=k + L, ragged=ragged)
    ex = fe.ORBextractor(1000, 1.2, 8)
    base = textured_frame(640, 480, seed=4)
    frames = np.stack([base, shifted_frame(base, 3, -2, seed=1), np.zeros_like(base), shifted_frame(base, -4, 1, seed=2)])
    kps, desc, counts = ex.extract_batch(frames)
    ex.close()
    assert counts[2] == 0 and counts[0] > 500
    counts = counts.copy()
    counts[3] = 617   # frames of different counts in one launch
    F, cap = desc.shape[0], desc.shape[1]
    v = B.Vocabulary(voc)
    d_desc = torch.from_numpy(np.ascontiguousarray(desc)).to(dev)
    d_cnt = torch.from_numpy(counts).to(dev)
    d_leaf = torch.zeros(F * cap, dtype=torch.int32, device=dev)
    d_node = torch.zeros(F * cap, dtype=torch.int32, device=dev)
    d_ids = torch.full((F, cap), -7, dtype=torch.int32, device=dev)
    d_ptr = torch.full((F, cap + 1), -7, dtype=torch.int32, device=dev)
    d_items = torch.full((F, cap), -7, dtype=torch.int32, device=dev)
    d_n = torch.full((F,), -7, dtype=torch.int32, device=dev)
    s = torch.cuda.Stream(device=dev)
    torch.cuda.synchronize()
    v.descend_device(d_desc.data_ptr(), F * cap, levelsup, d_leaf.data_ptr(), d_node.data_ptr(), s.cuda_stream)
    B.feature_vector_device(v, F, d_leaf.data_ptr(), d_node.data_ptr(), d_cnt.data_ptr(), cap, d_ids.data_ptr(), d_ptr.data_ptr(),
                            d_items.data_ptr(), d_n.data_ptr(), s.cuda_stream)
    s.synchronize()
    ids, ptr, items, n = (t.cpu().numpy() for t in (d_ids, d_ptr, d_items, d_n))
    node, leaf = d_node.cpu().numpy().reshape(F, cap), d_leaf.cpu().numpy().reshape(F, cap)
    stopped = 0
    for f in range(F):
        c = int(counts[f])
        got = _unpack_fv(ids, ptr, items, n, f)
        # features of stopped words (weight 0) are in no node
        kept = np.nonzero(voc["weight"][leaf[f, :c]] > 0)[0].astype(np.int32)
        stopped += c - len(kept)
        fid, fptr, fit = M.feature_vector(node[f, kept])
        assert _fv_equal(got, (fid, fptr, kept[fit])), f
        assert _fv_equal(got, v.transform(desc[f, :c], levelsup)[1]), f
        assert _fv_equal(got, O.bow_transform(voc, desc[f, :c], levelsup)[1]), f
        if c == 0:
            assert n[f] == 0 and ptr[f, 0] == 0
        else:
            assert np.all(np.diff(got[0]) > 0)
    if levelsup >= L:   # every node id is the root's: one node per non-empty frame
        assert list(n) == [1, 1, 0, 1]
    else:
        assert n[0] > 5
    assert stopped > 0   # the vocabulary has stopped words, so the weight test is exercised
    v.close()


# ---------------------------------------------------------------------------------------------------------------------
# 2. Batched SearchByBoW against the oracle
# ---------------------------------------------------------------------------------------------------------------------
def _bow_store(seed, cap=1600, nkf=30):
    """A frame store for SearchByBoW: frame 0 is the current frame, frames 1..nkf keyframes that saw subsets of the same
    features (noisy descriptors, rotated angles), frame nkf+1 has no features, frames nkf+2 / nkf+3 keep every feature in one
    node.  Node of a feature = a coarse function of a descriptor byte (noisy copies mostly share it); some features of frame
    0 sit in a node no keyframe has."""
    rng = np.random.default_rng(seed)
    nbase = 1500
    d0 = random_descriptors(nbase, seed)
    a0 = rng.uniform(0, 360, nbase).astype(np.float32)
    F = nkf + 4
    desc = np.zeros((F, cap, 32), np.uint8)
    ang = np.zeros((F, cap), np.float32)
    counts = np.zeros(F, np.int32)
    nodes = [None] * F

    def put(f, sel, flip, one_node=False):
        n = len(sel)
        desc[f, :n] = noisy_copies(d0[sel], flip, 1000 * seed + f)
        ang[f, :n] = ((a0[sel] + rng.normal(7, 4, n)) % 360).astype(np.float32)
        counts[f] = n
        nodes[f] = np.zeros(n, np.int32) if one_node else (desc[f, :n, 0].astype(np.int32) >> 3) * 3 + 11

    put(0, rng.permutation(nbase)[:1400], 0.05)
    nodes[0][rng.random(1400) < 0.05] = 9999   # a node only one side has
    for f in range(1, nkf + 1):
        put(f, rng.permutation(nbase)[:int(rng.integers(300, 1500))], 0.04)
    counts[nkf + 1] = 0
    nodes[nkf + 1] = np.zeros(0, np.int32)
    put(nkf + 2, rng.permutation(nbase)[:1400], 0.05, one_node=True)
    put(nkf + 3, rng.permutation(nbase)[:1300], 0.05, one_node=True)
    valid = (rng.random((F, cap)) < 0.85).astype(np.uint8)
    kps = np.zeros((F, cap), fe.KP_DTYPE)
    kps["angle"] = ang
    fvs = [M.feature_vector(nd) for nd in nodes]
    return kps, desc, counts, valid, fvs


def _jobs(nkf, variant):
    E, U1, U2 = nkf + 1, nkf + 2, nkf + 3
    if variant == 0:   # relocalisation: every keyframe against the current frame (side 2 shared)
        jobs = [(f, 0) for f in range(1, nkf + 1)]
    else:              # loop closing: one keyframe against every candidate (side 1 shared)
        jobs = [(0, f) for f in range(1, nkf + 1)]
    jobs += [jobs[3], (E, 0), (1, E), (E, E), (U1, U2), (U2, U1)]   # duplicated job, empty FeatureVectors, one node
    return np.array(jobs, np.int32)


def _run_device(m, variant, kps, desc, counts, valid, fv_slots, jobs):
    torch, dev = _torch()
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev)
    F, cap = desc.shape[:2]
    d_kps, d_desc, d_cnt, d_valid = t(kps.view(np.uint8).reshape(F, cap, 28)), t(desc), t(counts), t(valid)
    d_ids, d_ptr, d_items, d_n = (t(a) for a in fv_slots)
    d_i1, d_i2 = t(jobs[:, 0]), t(jobs[:, 1])
    nj = len(jobs)
    d_out = torch.full((nj, cap), -9, dtype=torch.int32, device=dev)
    d_nm = torch.full((nj,), -9, dtype=torch.int32, device=dev)
    s = torch.cuda.Stream(device=dev)
    torch.cuda.synchronize()
    M.search_by_bow_device(m, variant, nj, d_kps.data_ptr(), d_desc.data_ptr(), d_cnt.data_ptr(), cap, d_ids.data_ptr(), d_ptr.data_ptr(),
                           d_items.data_ptr(), d_n.data_ptr(), d_valid.data_ptr(), d_i1.data_ptr(), d_i2.data_ptr(), d_out.data_ptr(),
                           d_nm.data_ptr(), s.cuda_stream)
    s.synchronize()
    return d_out.cpu().numpy(), d_nm.cpu().numpy()


def _oracle_job(variant, kps, desc, counts, valid, fvs, f1, f2, nnr, ori):
    n1, n2 = counts[f1], counts[f2]
    return O.search_by_bow(variant, desc[f1, :n1], valid[f1, :n1], kps[f1, :n1]["angle"], fvs[f1], desc[f2, :n2], valid[f2, :n2],
                           kps[f2, :n2]["angle"], fvs[f2], nnratio=nnr, check_orientation=ori)


@pytest.mark.parametrize("seed", [3, 17, 40])
def test_search_by_bow_device_matches_oracle(gpu_required, seed):
    nkf = 30
    kps, desc, counts, valid, fvs = _bow_store(seed, nkf=nkf)
    slots = _pack_fvs(fvs, desc.shape[1])
    for variant in (0, 1):
        jobs = _jobs(nkf, variant)
        assert len(jobs) >= 32
        for nnr, ori in ((0.75, True), (0.6, False)):
            m = fe.ORBmatcher(nnr, ori)
            out, nm = _run_device(m, variant, kps, desc, counts, valid, slots, jobs)
            m.sync()
            one_node = 0
            for j, (f1, f2) in enumerate(jobs):
                n_o, out_o = _oracle_job(variant, kps, desc, counts, valid, fvs, f1, f2, nnr, ori)
                nout = counts[f2] if variant == 0 else counts[f1]
                assert nm[j] == n_o and np.array_equal(out[j, :nout], out_o), (variant, nnr, ori, j, f1, f2)
                if f1 >= nkf + 2 and f2 >= nkf + 2:
                    one_node += n_o
            assert nm[:nkf].sum() > 300 * 4 and one_node > 300, (variant, nnr, ori)
            assert nm[nkf] == nm[3]
            m.close()


# ---------------------------------------------------------------------------------------------------------------------
# 3. The whole chain on the device
# ---------------------------------------------------------------------------------------------------------------------
def test_device_chain_extract_descend_fv_search(gpu_required):
    """orbfe_extract_batch_device -> orbfe_bow_descend_device -> orbfe_feature_vector_device -> orbfe_search_by_bow_device with
    no host copy in between; equal to the host orbfe_search_by_bow on the downloaded arrays and to the oracle."""
    torch, dev = _torch()
    W, H, NF, levelsup = 640, 480, 1000, 3
    base = textured_frame(W, H, seed=11)
    frames = np.stack([base] + [shifted_frame(base, 2 * i, -i, seed=i) for i in range(1, 6)])
    Bn = len(frames)
    voc = random_vocabulary(10, 4, seed=6)
    v = B.Vocabulary(voc)
    ex = fe.ORBextractor(NF, 1.2, 8)
    rng = np.random.default_rng(2)
    d_frames = torch.from_numpy(frames).to(dev)
    d_valid = torch.from_numpy((rng.random((Bn, NF)) < 0.9).astype(np.uint8)).to(dev)   # the caller's map-point flags
    d_kps = torch.zeros((Bn, NF, 28), dtype=torch.uint8, device=dev)
    d_desc = torch.zeros((Bn, NF, 32), dtype=torch.uint8, device=dev)
    d_cnt = torch.zeros((Bn,), dtype=torch.int32, device=dev)
    d_leaf = torch.zeros(Bn * NF, dtype=torch.int32, device=dev)
    d_node = torch.zeros(Bn * NF, dtype=torch.int32, device=dev)
    d_ids = torch.zeros((Bn, NF), dtype=torch.int32, device=dev)
    d_ptr = torch.zeros((Bn, NF + 1), dtype=torch.int32, device=dev)
    d_items = torch.zeros((Bn, NF), dtype=torch.int32, device=dev)
    d_n = torch.zeros((Bn,), dtype=torch.int32, device=dev)
    jobs = {0: np.array([(f, 0) for f in range(1, Bn)], np.int32), 1: np.array([(0, f) for f in range(1, Bn)] + [(2, 3)], np.int32)}
    d_jobs = {k: (torch.from_numpy(j[:, 0].copy()).to(dev), torch.from_numpy(j[:, 1].copy()).to(dev)) for k, j in jobs.items()}
    d_out = {k: torch.zeros((len(j), NF), dtype=torch.int32, device=dev) for k, j in jobs.items()}
    d_nm = {k: torch.zeros(len(j), dtype=torch.int32, device=dev) for k, j in jobs.items()}
    m = fe.ORBmatcher(0.75, True)
    s = torch.cuda.Stream(device=dev)
    torch.cuda.synchronize()
    ex.extract_batch_device(d_frames.data_ptr(), W, H, W, W * H, Bn, d_kps.data_ptr(), d_desc.data_ptr(), d_cnt.data_ptr(), s.cuda_stream)
    v.descend_device(d_desc.data_ptr(), Bn * NF, levelsup, d_leaf.data_ptr(), d_node.data_ptr(), s.cuda_stream)
    B.feature_vector_device(v, Bn, d_leaf.data_ptr(), d_node.data_ptr(), d_cnt.data_ptr(), NF, d_ids.data_ptr(), d_ptr.data_ptr(),
                            d_items.data_ptr(), d_n.data_ptr(), s.cuda_stream)
    for variant in (0, 1):
        d_i1, d_i2 = d_jobs[variant]
        M.search_by_bow_device(m, variant, len(jobs[variant]), d_kps.data_ptr(), d_desc.data_ptr(), d_cnt.data_ptr(), NF, d_ids.data_ptr(),
                               d_ptr.data_ptr(), d_items.data_ptr(), d_n.data_ptr(), d_valid.data_ptr(), d_i1.data_ptr(),
                               d_i2.data_ptr(), d_out[variant].data_ptr(), d_nm[variant].data_ptr(), s.cuda_stream)
    s.synchronize()
    m.sync()
    kps = d_kps.cpu().numpy().view(fe.KP_DTYPE).reshape(Bn, NF)
    desc, counts, valid = d_desc.cpu().numpy(), d_cnt.cpu().numpy(), d_valid.cpu().numpy()
    ids, ptr, items, n = (t.cpu().numpy() for t in (d_ids, d_ptr, d_items, d_n))
    fvs = [_unpack_fv(ids, ptr, items, n, f) for f in range(Bn)]
    for f in range(Bn):
        assert _fv_equal(fvs[f], O.bow_transform(voc, desc[f, :counts[f]], levelsup)[1])
    total = 0
    for variant in (0, 1):
        out, nm = d_out[variant].cpu().numpy(), d_nm[variant].cpu().numpy()
        for j, (f1, f2) in enumerate(jobs[variant]):
            n1, n2 = counts[f1], counts[f2]
            nout = n2 if variant == 0 else n1
            args = (variant, desc[f1, :n1], valid[f1, :n1], kps[f1, :n1]["angle"], fvs[f1], desc[f2, :n2], valid[f2, :n2],
                    kps[f2, :n2]["angle"], fvs[f2])
            n_h, out_h = M.search_by_bow(m, *args)
            n_o, out_o = O.search_by_bow(*args, nnratio=0.75, check_orientation=True)
            assert nm[j] == n_h == n_o, (variant, j)
            assert np.array_equal(out[j, :nout], out_h) and np.array_equal(out_h, out_o), (variant, j)
            total += int(nm[j])
    assert total > 100
    ex.close(); v.close(); m.close()


# ---------------------------------------------------------------------------------------------------------------------
# 4. A malformed FeatureVector is bounds-checked
# ---------------------------------------------------------------------------------------------------------------------
def test_out_of_range_item_fails_only_its_job(gpu_required):
    nkf = 30
    kps, desc, counts, valid, fvs = _bow_store(5, nkf=nkf)
    cap = desc.shape[1]
    ids, ptr, items, n = _pack_fvs(fvs, cap)
    bad_frame = 7
    items = items.copy()
    items[bad_frame, :counts[bad_frame]] = counts[bad_frame] + 5   # every feature index of the frame is out of range
    jobs = _jobs(nkf, 0)
    m = fe.ORBmatcher(0.75, True)
    out, nm = _run_device(m, 0, kps, desc, counts, valid, (ids, ptr, items, n), jobs)
    with pytest.raises(fe.OrbfeError) as e:
        m.sync()
    assert e.value.code == fe.ORBFE_ERR_ARG
    m.sync()   # the flag is cleared by the report
    checked = 0
    for j, (f1, f2) in enumerate(jobs):
        if f1 == bad_frame or f2 == bad_frame:
            assert nm[j] == -1
            continue
        n_o, out_o = _oracle_job(0, kps, desc, counts, valid, fvs, f1, f2, 0.75, True)
        assert nm[j] == n_o and np.array_equal(out[j, :counts[f2]], out_o), j
        checked += 1
    assert checked >= 32
    m.close()
