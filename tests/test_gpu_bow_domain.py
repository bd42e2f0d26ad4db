"""The BoW chain and the Hamming kernels on the scenes of tests/bow_domain_scenes.py, bit for bit against the oracle: vocabulary
descent on tie trees and on ORBvoc's shape, FeatureVectors at every chunk and shared-memory size, SearchByBoW and
SearchForTriangulation on their rule boundaries and at cap 65535, ComputeDistinctiveDescriptors on lane edges, and the
Hamming primitives at every distance and past 65535 queries."""
import numpy as np
import pytest

import bow_domain_scenes as S
import oracle as O
import orb_slam_b200 as fe
from orb_slam_b200 import bow as B
from orb_slam_b200 import matching as M

pytestmark = pytest.mark.gpu


def _torch():
    import torch
    return torch, torch.device("cuda", 0)


def _dev(a):
    torch, dev = _torch()
    return torch.from_numpy(np.ascontiguousarray(a)).to(dev)


# ---- Hamming primitives ----------------------------------------------------------------------------------------------------
def test_hamming_every_distance_and_placement(gpu_required):
    q, t, d = S.distance_set()
    m = fe.ORBmatcher()
    D = m.hamming_dense(q, t)
    assert np.array_equal(np.diagonal(D), d)
    assert np.array_equal(D, S.hamming(q[:, None, :], t[None, :, :]))
    # CSR: the diagonal pairs plus rows longer than 32, empty rows between non-empty ones, nq = 771 (not a multiple of 8)
    rng = np.random.default_rng(1)
    rows = [np.array([i] + list(rng.choice(len(t), int(rng.choice([0, 3, 33, 70])), replace=False)), np.int32)
            if i % 5 else np.zeros(0, np.int32) for i in range(len(q))]
    ptr = np.concatenate([[0], np.cumsum([len(r) for r in rows])]).astype(np.int32)
    out = m.hamming_csr(q, t, ptr, np.concatenate(rows).astype(np.int32))
    assert np.array_equal(out, np.concatenate([D[i, r] for i, r in enumerate(rows)]))
    # the CSA popcount of knn2: one group per query, holding only its partner
    best, idx, second = m.knn2_groups(q, t, 1)
    assert np.array_equal(np.diagonal(best), d) and np.all(second == 65535)
    m.close()


@pytest.mark.parametrize("nq,nt", [(65536, 3), (70000, 5), (5, 64 * 256 + 77)])
def test_hamming_dense_past_the_grid_limits(gpu_required, nq, nt):
    rng = np.random.default_rng(nq)
    q = rng.integers(0, 256, (nq, 32), dtype=np.uint8)
    t = rng.integers(0, 256, (nt, 32), dtype=np.uint8)
    m = fe.ORBmatcher()
    D = m.hamming_dense(q, t)
    assert np.array_equal(D, S.hamming(q[:, None, :], t[None, :, :]))
    m.close()


@pytest.mark.parametrize("g", [1, 127, 128, 129, 255, 256, 1000])
def test_knn2_groups_chunk_edges_and_ties(gpu_required, g):
    m = fe.ORBmatcher()
    for nq in (1, 255, 256, 257, 1000):
        q, db, planted = S.knn2_scene(g, nq, seed=g + nq)
        best, idx, second = m.knn2_groups(q, db, g)
        for grp in range(2):
            bd, bi, sd = O.knn2(q, db[grp * g:(grp + 1) * g])
            assert np.array_equal(best[grp], bd) and np.array_equal(idx[grp], bi), (g, nq, grp)
            assert np.array_equal(second[grp], np.minimum(sd, 65535)), (g, nq, grp)
        for qi, grp, pos in planted:
            assert idx[grp, qi] == pos[0] and best[grp, qi] == second[grp, qi] == 10, (g, nq, pos)
    m.close()


# ---- vocabulary descent ----------------------------------------------------------------------------------------------------
LEVELSUPS = lambda L: sorted({0, 1, 4, L - 1, L, L + 1, 1000})


def _descend_device(v, q, levelsup):
    torch, dev = _torch()
    n = len(q)
    d_leaf = torch.full((n,), -9, dtype=torch.int32, device=dev)
    d_node = torch.full((n,), -9, dtype=torch.int32, device=dev)
    d_q = _dev(q)
    torch.cuda.synchronize()
    v.descend_device(d_q.data_ptr(), n, levelsup, d_leaf.data_ptr(), d_node.data_ptr())
    torch.cuda.synchronize()
    return d_leaf.cpu().numpy(), d_node.cpu().numpy()


@pytest.mark.parametrize("k,L", [(1, 6), (2, 6), (31, 4), (32, 4), (33, 4), (64, 3), (100, 3), (100, 2)])
def test_descent_on_tie_trees(gpu_required, k, L):
    voc = S.tie_vocabulary(k, L, seed=k)
    q, labels = S.tie_queries(voc, seed=k)
    v = B.Vocabulary(voc)
    for levelsup in LEVELSUPS(L):
        want = O.bow_descend(voc, q, levelsup)
        got = v.descend(q, levelsup)
        assert np.array_equal(got[0], want[0]) and np.array_equal(got[1], want[1]), (k, L, levelsup)
        got = _descend_device(v, q, levelsup)
        assert np.array_equal(got[0], want[0]) and np.array_equal(got[1], want[1]), (k, L, levelsup)
        for n in (1, 7, 9):   # not multiples of the 8 warps of a block
            got = v.descend(q[:n], levelsup)
            assert np.array_equal(got[0], want[0][:n]) and np.array_equal(got[1], want[1][:n]), (k, L, levelsup, n)
    v.close()


def test_descent_orbvoc_shape(gpu_required):
    voc = S.orbvoc_shape_vocabulary()
    q, _ = S.orbvoc_queries(voc, 64)
    v = B.Vocabulary(voc)
    for levelsup in (0, 1, 4, 5, 6, 7):
        want = O.bow_descend(voc, q, levelsup)
        got = _descend_device(v, q, levelsup)
        assert np.array_equal(got[0], want[0]) and np.array_equal(got[1], want[1]), levelsup
    assert (want[0] >= 1 << 20).sum() >= 8
    v.close()


# ---- FeatureVector ---------------------------------------------------------------------------------------------------------
_FV_VOC = None


def _fv_voc():
    global _FV_VOC
    if _FV_VOC is None:
        voc = S.tie_vocabulary(8, 2, seed=3)   # 25 nodes; the internal nodes and one leaf have weight 0
        _FV_VOC = (voc, B.Vocabulary(voc))
    return _FV_VOC


def _fv_device(v, leaf, node, counts, cap):
    torch, dev = _torch()
    F = len(counts)
    d_ids = torch.full((F, cap), -7, dtype=torch.int32, device=dev)
    d_ptr = torch.full((F, cap + 1), -7, dtype=torch.int32, device=dev)
    d_items = torch.full((F, cap), -7, dtype=torch.int32, device=dev)
    d_n = torch.full((F,), -7, dtype=torch.int32, device=dev)
    d_leaf, d_node, d_cnt = _dev(leaf), _dev(node), _dev(counts)
    torch.cuda.synchronize()
    B.feature_vector_device(v, F, d_leaf.data_ptr(), d_node.data_ptr(), d_cnt.data_ptr(), cap, d_ids.data_ptr(), d_ptr.data_ptr(),
                            d_items.data_ptr(), d_n.data_ptr())
    torch.cuda.synchronize()
    return tuple(t.cpu().numpy() for t in (d_ids, d_ptr, d_items, d_n))


@pytest.mark.parametrize("cap", S.FV_CAPS)
def test_feature_vector_every_chunk_and_smem_size(gpu_required, cap):
    voc, v = _fv_voc()
    live = voc["weight"] > 0
    leaf, node, counts = S.fv_frames(cap, len(live), live, seed=cap)
    ids, ptr, items, n = _fv_device(v, leaf, node, counts, cap)
    for f in range(len(counts)):
        wi, wp, wt = S.fv_numpy(leaf[f], node[f], counts[f], cap, live)
        k = len(wi)
        assert n[f] == k and np.array_equal(ids[f, :k], wi) and np.array_equal(ptr[f, :k + 1], wp), (cap, f)
        assert np.array_equal(items[f, :wp[-1]], wt), (cap, f)
        # nothing is written past the FeatureVector
        assert np.all(ids[f, k:] == -7) and np.all(ptr[f, k + 1:] == -7) and np.all(items[f, wp[-1]:] == -7), (cap, f)


def test_feature_vector_refuses_cap_16385(gpu_required):
    torch, dev = _torch()
    voc, v = _fv_voc()
    cap = 16385
    d = [torch.full((2, cap + 1), -7, dtype=torch.int32, device=dev) for _ in range(6)]
    d_cnt = torch.full((2,), 3, dtype=torch.int32, device=dev)
    torch.cuda.synchronize()
    with pytest.raises(fe.OrbfeError) as e:
        B.feature_vector_device(v, 2, d[0].data_ptr(), d[1].data_ptr(), d_cnt.data_ptr(), cap, d[2].data_ptr(), d[3].data_ptr(),
                                d[4].data_ptr(), d[5].data_ptr())
    assert e.value.code == fe.ORBFE_ERR_UNSUPPORTED
    torch.cuda.synchronize()
    assert all(bool((x == -7).all()) for x in d[2:])


_CHAIN = None


def _chain_voc():
    global _CHAIN
    if _CHAIN is None:
        voc = S.tie_vocabulary(40, 4, seed=9)   # 601 nodes; the leaf of the "distance 0" query is stopped
        _CHAIN = (voc, B.Vocabulary(voc))
    return _CHAIN


@pytest.mark.parametrize("cap", S.FV_CAPS)
def test_feature_vector_chain_against_the_oracle(gpu_required, cap):
    """Descriptors -> orbfe_bow_descend_device -> orbfe_feature_vector_device on one stream, with no host copy in between, at
    every cap of the sweep, against the oracle's DBoW2 transform of the same descriptors."""
    torch, dev = _torch()
    voc, v = _chain_voc()
    rng = np.random.default_rng(cap)
    q, _ = S.tie_queries(voc, seed=9)
    F = 4
    desc = np.stack([q[rng.integers(0, len(q), cap)] for _ in range(F)])
    desc[1, ::3] = rng.integers(0, 256, (len(desc[1, ::3]), 32), dtype=np.uint8)
    counts = np.array([cap, (cap + 1) // 2, 0, min(cap, 1025)], np.int32)
    d_desc, d_cnt = _dev(desc), _dev(counts)
    s = torch.cuda.Stream(device=dev)
    for levelsup in (0, 2, 4):
        d_leaf = torch.full((F * cap,), -9, dtype=torch.int32, device=dev)
        d_node = torch.full((F * cap,), -9, dtype=torch.int32, device=dev)
        d_ids = torch.full((F, cap), -7, dtype=torch.int32, device=dev)
        d_ptr = torch.full((F, cap + 1), -7, dtype=torch.int32, device=dev)
        d_items = torch.full((F, cap), -7, dtype=torch.int32, device=dev)
        d_n = torch.full((F,), -7, dtype=torch.int32, device=dev)
        torch.cuda.synchronize()   # the uploads and fills above ran on torch's stream
        v.descend_device(d_desc.data_ptr(), F * cap, levelsup, d_leaf.data_ptr(), d_node.data_ptr(), s.cuda_stream)
        B.feature_vector_device(v, F, d_leaf.data_ptr(), d_node.data_ptr(), d_cnt.data_ptr(), cap, d_ids.data_ptr(), d_ptr.data_ptr(),
                                d_items.data_ptr(), d_n.data_ptr(), s.cuda_stream)
        s.synchronize()
        ids, ptr, items, n = (t.cpu().numpy() for t in (d_ids, d_ptr, d_items, d_n))
        for f in range(F):
            k = int(n[f])
            got = (ids[f, :k], ptr[f, :k + 1], items[f, :ptr[f, k]])
            want = O.bow_transform(voc, desc[f, :counts[f]], levelsup)[1]
            assert all(np.array_equal(a, b) for a, b in zip(got, want)), (cap, levelsup, f)


# ---- frame stores for the matchers ------------------------------------------------------------------------------------------
def _store(pairs):
    """Stack (f1, f2) Frame pairs into one frame store; job j = (2j, 2j + 1)."""
    frames = [f for p in pairs for f in p]
    cap = max(len(f.desc) for f in frames)
    F = len(frames)
    kps = np.zeros((F, cap), S.KP_DTYPE)
    desc = np.zeros((F, cap, 32), np.uint8)
    flag = np.zeros((F, cap), np.uint8)
    ids, items = np.zeros((F, cap), np.int32), np.zeros((F, cap), np.int32)
    ptr, n = np.zeros((F, cap + 1), np.int32), np.zeros(F, np.int32)
    counts = np.zeros(F, np.int32)
    for k, f in enumerate(frames):
        c = len(f.desc)
        kps[k, :c], desc[k, :c], flag[k, :c], counts[k] = f.kps, f.desc, f.flag, c
        i, p, t = f.fv()
        ids[k, :len(i)], ptr[k, :len(p)], items[k, :len(t)], n[k] = i, p, t, len(i)
    return dict(kps=kps, desc=desc, flag=flag, counts=counts, cap=cap, slots=(ids, ptr, items, n))


def _bow_device(st, variant, jobs, nnratio, ori):
    torch, dev = _torch()
    jobs = np.asarray(jobs, np.int32)
    F, cap = st["desc"].shape[:2]
    d_kps = _dev(st["kps"].view(np.uint8).reshape(F, cap, 28))
    d_desc, d_cnt, d_flag = _dev(st["desc"]), _dev(st["counts"]), _dev(st["flag"])
    d_ids, d_ptr, d_items, d_n = (_dev(a) for a in st["slots"])
    d_i1, d_i2 = _dev(jobs[:, 0].copy()), _dev(jobs[:, 1].copy())
    d_out = torch.full((len(jobs), cap), -9, dtype=torch.int32, device=dev)
    d_nm = torch.full((len(jobs),), -9, dtype=torch.int32, device=dev)
    m = fe.ORBmatcher(nnratio, ori)
    torch.cuda.synchronize()
    M.search_by_bow_device(m, variant, len(jobs), d_kps.data_ptr(), d_desc.data_ptr(), d_cnt.data_ptr(), cap, d_ids.data_ptr(),
                           d_ptr.data_ptr(), d_items.data_ptr(), d_n.data_ptr(), d_flag.data_ptr(), d_i1.data_ptr(), d_i2.data_ptr(),
                           d_out.data_ptr(), d_nm.data_ptr())
    torch.cuda.synchronize()
    m.sync()
    return m, d_out.cpu().numpy(), d_nm.cpu().numpy()


def _bow_check(st, frames, variant, jobs, nnratio, ori, host=False):
    m, out, nm = _bow_device(st, variant, jobs, nnratio, ori)
    rows = []
    for j, (a, b) in enumerate(jobs):
        f1, f2 = frames[a], frames[b]
        args = (variant, f1.desc, f1.flag, f1.kps["angle"], f1.fv(), f2.desc, f2.flag, f2.kps["angle"], f2.fv())
        n_o, o_o = O.search_by_bow(*args, nnratio=nnratio, check_orientation=ori)
        nout = len(f2.desc) if variant == 0 else len(f1.desc)
        assert nm[j] == n_o and np.array_equal(out[j, :nout], o_o), (variant, nnratio, ori, j)
        if host:
            n_h, o_h = M.search_by_bow(m, *args)
            assert n_h == n_o and np.array_equal(o_h, o_o), (variant, nnratio, ori, j)
        rows.append(out[j, :nout])
    m.close()
    return rows


@pytest.mark.parametrize("variant", [0, 1])
def test_search_by_bow_rule_boundaries(gpu_required, variant):
    f1, f2, E = S.bow_boundary_pair()
    st = _store([(f1, f2)])
    frames = [f1, f2]
    for r in S.BOW_RATIOS:
        (row,) = _bow_check(st, frames, variant, [(0, 1)], r, False, host=True)
        for lab, i1, i2 in E.applicable(variant=variant, nnratio=r):
            assert S.match_of(variant, row, i1) == i2, (variant, r, lab)
    # 300 jobs in one launch: duplicates, f1 == f2 and the reversed pair
    jobs = [(0, 1)] * 150 + [(0, 0), (1, 1), (1, 0)] * 50
    _bow_check(st, frames, variant, jobs, 0.75, True)


@pytest.mark.parametrize("variant", [0, 1])
def test_search_by_bow_rotation_histogram(gpu_required, variant):
    jobs = S.rotation_jobs()
    pairs = [S.rotation_pair(mt, j)[:2] for j, (_, mt, _) in enumerate(jobs)]
    kept_pairs = [S.rotation_pair(mt, j)[2] for j, (_, mt, _) in enumerate(jobs)]
    st = _store(pairs)
    frames = [f for p in pairs for f in p]
    jl = [(2 * j, 2 * j + 1) for j in range(len(pairs))]
    for ori in (True, False):
        rows = _bow_check(st, frames, variant, jl, 0.75, ori, host=ori)
        for (name, _, kept), pr, row in zip(jobs, kept_pairs, rows):
            got = [S.match_of(variant, row, i1) == i2 for i1, i2 in pr]
            assert got == (kept if ori else [True] * len(kept)), (name, ori)


def test_search_by_bow_cap_65535(gpu_required):
    f1, f2, E = S.big_pair("bow")
    st = _store([(f1, f2)])
    assert st["cap"] == 65535
    for variant in (0, 1):
        (row,) = _bow_check(st, [f1, f2], variant, [(0, 1)], 0.75, True)
        for lab, i1, i2 in E.applicable():
            assert S.match_of(variant, row, i1) == i2, (variant, lab)


# ---- SearchForTriangulation --------------------------------------------------------------------------------------------------
def _tri_check(st, frames, jobs, F12, sig2, ori, host=False):
    torch, dev = _torch()
    jobs = np.asarray(jobs, np.int32)
    F, cap = st["desc"].shape[:2]
    d_kps = _dev(st["kps"].view(np.uint8).reshape(F, cap, 28))
    d_desc, d_cnt, d_flag = _dev(st["desc"]), _dev(st["counts"]), _dev(st["flag"])
    d_ids, d_ptr, d_items, d_n = (_dev(a) for a in st["slots"])
    d_i1, d_i2, d_F = _dev(jobs[:, 0].copy()), _dev(jobs[:, 1].copy()), _dev(np.asarray(F12, np.float32))
    d_out = torch.full((len(jobs), cap), -9, dtype=torch.int32, device=dev)
    d_nm = torch.full((len(jobs),), -9, dtype=torch.int32, device=dev)
    m = fe.ORBmatcher(0.6, ori)
    torch.cuda.synchronize()
    M.search_for_triangulation_device(m, len(jobs), d_kps.data_ptr(), d_desc.data_ptr(), d_cnt.data_ptr(), cap, d_ids.data_ptr(),
                                      d_ptr.data_ptr(), d_items.data_ptr(), d_n.data_ptr(), d_flag.data_ptr(), d_i1.data_ptr(),
                                      d_i2.data_ptr(), d_F.data_ptr(), sig2, d_out.data_ptr(), d_nm.data_ptr())
    torch.cuda.synchronize()
    m.sync()
    out, nm = d_out.cpu().numpy(), d_nm.cpu().numpy()
    rows = []
    for j, (a, b) in enumerate(jobs):
        f1, f2 = frames[a], frames[b]
        args = (f1.kps, f1.desc, f1.flag, f1.fv(), f2.kps, f2.desc, f2.flag, f2.fv())
        n_o, m12 = O.search_for_triangulation(*args, F12[j], sig2, check_orientation=ori)
        assert nm[j] == n_o and np.array_equal(out[j, :len(f1.desc)], m12), (ori, j)
        if host:
            n_h, m12_h = M.search_for_triangulation(m, *args, F12[j], sig2)
            assert n_h == n_o and np.array_equal(m12_h, m12), (ori, j)
        rows.append(out[j, :len(f1.desc)])
    m.close()
    return rows


@pytest.mark.parametrize("nlevels", [8, 32])
def test_search_for_triangulation_rule_boundaries(gpu_required, nlevels):
    f1, f2, E, sig2 = S.tri_boundary_pair(nlevels=nlevels)
    st = _store([(f1, f2)])
    F12 = np.stack([S.F12_LINE_Y, np.zeros(9, np.float32), S.F12_LINE_Y]).astype(np.float32)
    for ori in (False, True):
        rows = _tri_check(st, [f1, f2], [(0, 1), (0, 1), (1, 0)], F12, sig2, ori, host=True)
        if not ori:
            for lab, i1, i2 in E.applicable():
                assert rows[0][i1] == i2, lab
        assert np.all(rows[1] == -1)   # F12 = 0: den == 0 rejects everything


def test_search_for_triangulation_rotation_histogram(gpu_required):
    jobs = S.rotation_jobs()
    built = [S.rotation_pair(mt, j, kind="tri") for j, (_, mt, _) in enumerate(jobs)]
    st = _store([b[:2] for b in built])
    frames = [f for b in built for f in b[:2]]
    jl = [(2 * j, 2 * j + 1) for j in range(len(built))]
    F12 = np.repeat(S.F12_LINE_Y[None, :], len(jl), axis=0)
    rows = _tri_check(st, frames, jl, F12, S.sigma2(8), True, host=True)
    for (name, _, kept), b, row in zip(jobs, built, rows):
        assert [row[i1] == i2 for i1, i2 in b[2]] == kept, name


def test_search_for_triangulation_cap_65535(gpu_required):
    f1, f2, E = S.big_pair("tri")
    st = _store([(f1, f2)])
    F12 = S.F12_LINE_Y[None, :]
    for ori in (False, True):
        (row,) = _tri_check(st, [f1, f2], [(0, 1)], F12, S.sigma2(8), ori)
        for lab, i1, i2 in E.applicable():
            assert row[i1] == i2, (ori, lab)


# ---- ComputeDistinctiveDescriptors -------------------------------------------------------------------------------------------
def test_distinctive_descriptors_boundaries(gpu_required):
    torch, dev = _torch()
    groups = S.distinctive_groups()
    desc = np.concatenate([g for _, g in groups])
    ptr = np.concatenate([[0], np.cumsum([len(g) for _, g in groups])]).astype(np.int32)
    want = O.distinctive_descriptors(desc, ptr)
    m = fe.ORBmatcher()
    assert np.array_equal(B.distinctive_descriptors(m, desc, ptr), want)
    # device form: the observations scattered over a frame store in a shuffled slot order
    cap = 512
    nobs = len(desc)
    F = (nobs + cap - 1) // cap + 1
    rng = np.random.default_rng(0)
    slots = rng.permutation(F * cap)[:nobs].astype(np.int32)
    store = rng.integers(0, 256, (F * cap, 32), dtype=np.uint8)
    store[slots] = desc
    d_store, d_cnt, d_ptr, d_obs = _dev(store), _dev(np.full(F, cap, np.int32)), _dev(ptr), _dev(slots)
    ng = len(groups)
    d_best = torch.full((ng,), -9, dtype=torch.int32, device=dev)
    d_mp = torch.zeros((ng, 32), dtype=torch.uint8, device=dev)
    torch.cuda.synchronize()
    B.distinctive_descriptors_device(m, ng, d_store.data_ptr(), d_cnt.data_ptr(), F, cap, d_ptr.data_ptr(), d_obs.data_ptr(), nobs,
                                     d_best.data_ptr(), d_mp.data_ptr())
    torch.cuda.synchronize()
    m.sync()
    best, mp = d_best.cpu().numpy(), d_mp.cpu().numpy()
    assert np.array_equal(best, want)
    assert np.array_equal(mp, desc[ptr[:-1] + want])
    m.close()
