"""GPU parity of the SURVEY section 8(f) rows N2 (DBoW2 vocabulary transform) and N4 (batched
MapPoint::ComputeDistinctiveDescriptors): CUDA path through the C-ABI vs the oracle, bit-exact (ids and the float64
BowVector values, which are produced by the same additions in the same order)."""
import numpy as np
import pytest

import oracle as O
import orb_slam_b200 as fe
from orb_slam_b200 import bow as B
from orb_slam_b200.synth import random_descriptors, noisy_copies, random_vocabulary, random_keyframe_db

pytestmark = pytest.mark.gpu

MAX_CAP = 16384   # ORBFE_FV_MAX_CAP


def word_descriptors(voc, n, seed):
    """n noisy copies of the vocabulary's words, every 50th descriptor unrelated (seed >= 1)."""
    words = voc["node_desc"][voc["word_id"] >= 0]
    rng = np.random.default_rng(seed)
    desc = noisy_copies(words[rng.integers(0, len(words), n)], 0.1, seed + 4)
    desc[::50] = random_descriptors(len(desc[::50]), seed - 1)  # a few unrelated descriptors
    return desc


def modes(L):
    """(levelsup, weighting, norm): every weighting and norm once, levelsup from 0 to past the tree's depth."""
    return [(4, B.TF_IDF, B.NORM_L1), (2, B.TF, B.NORM_NONE), (0, B.IDF, B.NORM_L2), (L + 1, B.BINARY, B.NORM_L1)]


def assert_transform_equal(got, want, tag):
    (ids, vals), (fids, fptr, ffeat) = got
    (ids_o, vals_o), (fids_o, fptr_o, ffeat_o) = want
    assert np.array_equal(ids, ids_o) and np.array_equal(vals.view(np.uint64), vals_o.view(np.uint64)), tag
    assert np.array_equal(fids, fids_o) and np.array_equal(fptr, fptr_o) and np.array_equal(ffeat, ffeat_o), tag


@pytest.mark.parametrize("k,L,ragged,n", [(10, 4, False, 2000), (7, 3, True, 777), (40, 2, False, 500), (10, 5, True, 1500)])
def test_bow_transform_matches_oracle(gpu_required, k, L, ragged, n):
    voc = random_vocabulary(k, L, seed=k + L, ragged=ragged)
    desc = word_descriptors(voc, n, 5)
    for levelsup, weighting, norm in modes(L):
        v = B.Vocabulary(voc, weighting, norm)
        leaf, node = v.descend(desc, levelsup)
        leaf_o, node_o = O.bow_descend(voc, desc, levelsup)
        assert np.array_equal(leaf, leaf_o) and np.array_equal(node, node_o)
        got = v.transform(desc, levelsup)
        assert_transform_equal(got, O.bow_transform(voc, desc, levelsup, weighting, norm), (levelsup, weighting, norm))
        assert len(got[0][0]) > 10
        v.close()


def test_bow_transform_at_max_descriptors(gpu_required):
    """n = ORBFE_FV_MAX_CAP descriptors (128 KB of sort keys in shared memory per kernel) equals the oracle bit for bit for
    every weighting and norm; one more descriptor is ORBFE_ERR_UNSUPPORTED."""
    voc = random_vocabulary(10, 5, seed=15, ragged=True)
    desc = word_descriptors(voc, MAX_CAP + 1, 8)
    for levelsup, weighting, norm in modes(5):
        v = B.Vocabulary(voc, weighting, norm)
        got = v.transform(desc[:MAX_CAP], levelsup)
        assert_transform_equal(got, O.bow_transform(voc, desc[:MAX_CAP], levelsup, weighting, norm), (levelsup, weighting, norm))
        assert len(got[0][0]) > 1000
        v.close()
    v = B.Vocabulary(voc)
    with pytest.raises(fe.OrbfeError) as e:
        v.transform(desc, 4)
    assert e.value.code == fe.ORBFE_ERR_UNSUPPORTED
    v.close()


def test_bow_transform_writes_nothing_past_its_counts(gpu_required):
    """Output arrays of capacity n filled with a sentinel: orbfe_bow_transform writes the oracle's entries and leaves every
    entry past bow_ids / bow_vals[nw), fv_ids[nn), fv_ptr[nn] and fv_feats[fv_ptr[nn]) as it was."""
    import ctypes as C
    voc = random_vocabulary(10, 3, seed=4)
    L = B._bind()
    p = lambda a: a.ctypes.data_as(C.c_void_p)
    for n, seed in ((1, 1), (300, 2), (2000, 3), (5000, 4)):
        desc = word_descriptors(voc, n, seed)
        v = B.Vocabulary(voc)
        bow_ids, bow_vals = np.full(n, -5, np.int32), np.full(n, -5.0)
        fv_ids, fv_ptr, fv_feats = np.full(n, -5, np.int32), np.full(n + 1, -5, np.int32), np.full(n, -5, np.int32)
        nw, nn = C.c_int(-5), C.c_int(-5)
        assert L.orbfe_bow_transform(v.handle, p(desc), n, 1, C.byref(nw), p(bow_ids), p(bow_vals), C.byref(nn), p(fv_ids), p(fv_ptr),
                                     p(fv_feats)) == fe.ORBFE_OK
        nw, nn = nw.value, nn.value
        nf = fv_ptr[nn]
        assert_transform_equal(((bow_ids[:nw], bow_vals[:nw]), (fv_ids[:nn], fv_ptr[:nn + 1], fv_feats[:nf])), O.bow_transform(voc, desc, 1), n)
        assert (bow_ids[nw:] == -5).all() and (bow_vals[nw:] == -5.0).all() and (fv_ids[nn:] == -5).all(), n
        assert (fv_ptr[nn + 1:] == -5).all() and (fv_feats[nf:] == -5).all(), n
        if n > 1:
            assert nw < n and nn < n and nf < n, n   # some features fall on stopped words, several on one word
        v.close()


def test_bow_transform_from_several_threads(gpu_required):
    """Four threads call transform on one vocabulary, 50 calls each on descriptor sets of 1 to 2000 descriptors, all at
    once (ctypes releases the GIL): every result equals the oracle.  The first call is made at the largest size, so no
    call grows the staging block while others are in flight."""
    import threading
    voc = random_vocabulary(10, 4, seed=2)
    v = B.Vocabulary(voc)
    T, K, NMAX = 4, 50, 2000
    rng = np.random.default_rng(21)
    sizes = rng.integers(1, NMAX + 1, (T, K))
    sizes[:, 0] = NMAX
    sets = [[word_descriptors(voc, int(sizes[t, k]), 1000 * t + k + 1) for k in range(K)] for t in range(T)]
    want = [[O.bow_transform(voc, d, 4) for d in row] for row in sets]
    assert_transform_equal(v.transform(sets[0][0], 4), want[0][0], "warm-up")
    bad, start = [], threading.Barrier(T)

    def run(t):
        try:
            start.wait()
            for k in range(K):
                got = v.transform(sets[t][k], 4)
                try:
                    assert_transform_equal(got, want[t][k], (t, k))
                except AssertionError as e:
                    bad.append(e)
        except Exception as e:   # noqa: BLE001 -- reported below
            bad.append(e)

    threads = [threading.Thread(target=run, args=(t,)) for t in range(T)]
    for th in threads:
        th.start()
    for th in threads:
        th.join()
    assert not bad, bad[:3]
    v.close()


def test_bow_descend_device_chains_after_extraction(gpu_required):
    """Device-pointer form on the descriptors orbfe_extract_batch_device leaves in HBM (no host round trip)."""
    import torch
    from orb_slam_b200.synth import textured_frame
    voc = random_vocabulary(10, 4, seed=2)
    v = B.Vocabulary(voc)
    ex = fe.ORBextractor(1000, 1.2, 8)
    img = textured_frame(640, 480, seed=3)
    kps, desc = ex(img)
    dev = torch.device("cuda", 0)
    d_desc = torch.from_numpy(np.ascontiguousarray(desc)).to(dev)
    d_leaf = torch.zeros(len(desc), dtype=torch.int32, device=dev)
    d_node = torch.zeros(len(desc), dtype=torch.int32, device=dev)
    s = torch.cuda.Stream(device=dev)
    torch.cuda.synchronize()
    v.descend_device(d_desc.data_ptr(), len(desc), 4, d_leaf.data_ptr(), d_node.data_ptr(), s.cuda_stream)
    s.synchronize()
    leaf_o, node_o = O.bow_descend(voc, desc, 4)
    assert np.array_equal(d_leaf.cpu().numpy(), leaf_o) and np.array_equal(d_node.cpu().numpy(), node_o)
    ex.close()
    v.close()


def test_empty_and_error_cases(gpu_required):
    voc = random_vocabulary(3, 2, seed=0)
    v = B.Vocabulary(voc)
    (ids, vals), (fids, fptr, ffeat) = v.transform(np.zeros((0, 32), np.uint8))
    assert len(ids) == 0 and len(fids) == 0 and list(fptr) == [0]
    bad = dict(voc)
    bad["children"] = voc["children"].copy()
    bad["children"][0] = len(voc["word_id"]) + 5
    with pytest.raises(fe.OrbfeError):
        B.Vocabulary(bad)
    v.close()


def test_distinctive_descriptors_matches_oracle(gpu_required):
    rng = np.random.default_rng(12)
    groups, ptr = [], [0]
    for g in range(700):
        n = int(rng.integers(1, 60)) if g % 11 else int(rng.integers(0, 3))
        if g == 5:
            n = 400  # a long-lived map point
        base = random_descriptors(1, 1000 + g)
        groups.append(noisy_copies(np.repeat(base, n, axis=0), rng.uniform(0.01, 0.3), 5000 + g) if n else np.zeros((0, 32), np.uint8))
        ptr.append(ptr[-1] + n)
    desc = np.concatenate(groups)
    ptr = np.array(ptr, np.int32)
    m = fe.ORBmatcher(0.6, True)
    best = B.distinctive_descriptors(m, desc, ptr)
    best_o = O.distinctive_descriptors(desc, ptr)
    assert np.array_equal(best, best_o)
    assert (best >= 0).sum() > 600
    # empty batch
    assert len(B.distinctive_descriptors(m, np.zeros((0, 32), np.uint8), np.zeros(1, np.int32))) == 0
    m.close()


def test_keyframe_db_detect_matches_oracle(gpu_required):
    """N3: DetectLoopCandidates / DetectRelocalisationCandidates on arrays, CUDA scoring + host list logic vs the oracle's
    literal inverted-file walk: candidates in the same order, identical shared-word counts and float scores."""
    m = fe.ORBmatcher(0.75, True)
    for seed, nkf in ((0, 400), (1, 1500), (2, 60)):
        db = random_keyframe_db(nkf=nkf, nwords=8000, words_per_kf=300, seed=seed, loop_at=nkf // 5)
        for mode, ms in ((0, 0.0), (0, 0.03), (1, 0.0)):
            args = (db["q_ids"], db["q_vals"], db["kf_ptr"], db["db_ids"], db["db_vals"], db["connected"], db["covis_ptr"], db["covis"], ms)
            cand, common, score = B.db_detect(m, mode, *args)
            cand_o, common_o, score_o = O.bow_db_detect(mode, *args)
            assert np.array_equal(cand, cand_o), (seed, mode, ms)
            assert np.array_equal(common, common_o)
            assert np.array_equal(score.view(np.uint32), score_o.view(np.uint32))
            assert len(cand) > 0 and (nkf // 5 in cand or nkf // 5 + 1 in cand or nkf // 5 - 1 in cand)
    # a query that shares nothing
    db = random_keyframe_db(nkf=50, nwords=2000, words_per_kf=100, seed=5)
    cand, common, score = B.db_detect(m, 1, np.array([2001, 2002], np.int32), np.array([0.5, 0.5]), db["kf_ptr"], db["db_ids"], db["db_vals"],
                                      db["connected"], db["covis_ptr"], db["covis"], 0.0)
    assert len(cand) == 0 and common.sum() == 0
    m.close()
