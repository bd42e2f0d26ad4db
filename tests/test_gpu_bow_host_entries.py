"""The host-array SearchByBoW and SearchForTriangulation entries (orbfe_search_by_bow, orbfe_search_for_triangulation) on
inputs the scene tests do not reach: FeatureVector rows outside the item array, side-2 octaves outside the level range, the
65535-feature limit, variant 0 with valid2 = NULL, and FeatureVectors with empty nodes (more nodes than features).  Every
accepted call equals the oracle bit for bit, and a rejected call leaves the matcher usable."""
import ctypes as C

import numpy as np
import pytest

import bow_domain_scenes as S
import oracle as O
import orb_slam_b200 as fe
from orb_slam_b200 import matching as M

pytestmark = pytest.mark.gpu

MAX_LEVELS = 32   # ORBFE_MAX_LEVELS, include/orbfe.h


def _fv(node, ids):
    """FeatureVector over the node ids `ids` (ascending), empty nodes included."""
    cnt = [int((node == i).sum()) for i in ids]
    return (np.asarray(ids, np.int32), np.concatenate([[0], np.cumsum(cnt)]).astype(np.int32),
            np.argsort(node, kind="stable").astype(np.int32))


def _sparse_pair(seed=0):
    """Five features per side in FeatureVectors of 10 (side 1) and 12 (side 2) nodes, most of them empty.  Common nodes are
    empty on both sides, on either side or on neither; side 2's last two nodes are empty and not common."""
    rng = np.random.default_rng(seed)
    f1, f2 = S.Frame(5, 0, seed + 1), S.Frame(5, 0, seed + 2)
    f1.node[:] = [3, 3, 7, 9, 5]
    f2.node[:] = [3, 7, 7, 9, 8]
    for i2, i1, d in ((0, 0, 10), (1, 2, 20), (2, 2, 30), (3, 3, 5)):
        f2.desc[i2] = S.away(f1.desc[i1], d, rng)
    f2.kps["y"] = 0.0   # on the epipolar line of every side-1 feature for F12_LINE_Y
    return f1, f2, _fv(f1.node, range(10)), _fv(f2.node, range(12))


def _bow_args(variant, f1, f2, fv1, fv2):
    return (variant, f1.desc, f1.flag, f1.kps["angle"], fv1, f2.desc, f2.flag, f2.kps["angle"], fv2)


def _tri_args(f1, f2, fv1, fv2):
    return (f1.kps, f1.desc, f1.flag, fv1, f2.kps, f2.desc, f2.flag, fv2, S.F12_LINE_Y)


def _bow_equal(m, args):
    n_o, o_o = O.search_by_bow(*args, nnratio=m.mfNNratio, check_orientation=m.mbCheckOrientation)
    n_h, o_h = M.search_by_bow(m, *args)
    assert n_h == n_o and np.array_equal(o_h, o_o)
    return n_o


def _tri_equal(m, args, sig2):
    n_o, m12_o = O.search_for_triangulation(*args, sig2, check_orientation=m.mbCheckOrientation)
    n_h, m12_h = M.search_for_triangulation(m, *args, sig2)
    assert n_h == n_o and np.array_equal(m12_h, m12_o)
    return n_o


def _code(fn, *args):
    with pytest.raises(fe.OrbfeError) as e:
        fn(*args)
    return e.value.code


def _bad_rows(fv1, fv2):
    """(side, FeatureVector) pairs with one common node's row out of range: past ptr[nn] but inside the frame's slots (the
    item slots there are unused), past the slots, and starting below 0."""
    i2, p2, t2 = fv2
    past_items = p2.copy()
    past_items[10] = 9            # node 9, the last common node: [4, 9) with ptr[nn] = 5 and 12 slots
    past_slots = p2.copy()
    past_slots[4] = len(t2) + 100
    i1, p1, t1 = fv1
    negative = p1.copy()
    negative[0] = -1
    return [(2, (i2, past_items, t2)), (2, (i2, past_slots, t2)), (1, (i1, negative, t1))]


@pytest.mark.parametrize("variant", [0, 1])
def test_search_by_bow_rejects_rows_outside_the_items(gpu_required, variant):
    f1, f2, fv1, fv2 = _sparse_pair()
    f1.flag[:] = 1
    f2.flag[:] = 1
    m = fe.ORBmatcher(0.75, True)
    assert _bow_equal(m, _bow_args(variant, f1, f2, fv1, fv2)) > 0
    for side, bad in _bad_rows(fv1, fv2):
        args = _bow_args(variant, f1, f2, bad if side == 1 else fv1, bad if side == 2 else fv2)
        assert _code(M.search_by_bow, m, *args) == fe.ORBFE_ERR_ARG, side
        assert _bow_equal(m, _bow_args(variant, f1, f2, fv1, fv2)) > 0
    m.close()


def test_search_for_triangulation_rejects_rows_and_octaves(gpu_required):
    f1, f2, fv1, fv2 = _sparse_pair()
    sig2 = S.sigma2(8)
    m = fe.ORBmatcher(0.6, True)
    assert _tri_equal(m, _tri_args(f1, f2, fv1, fv2), sig2) > 0
    for side, bad in _bad_rows(fv1, fv2):
        args = _tri_args(f1, f2, bad if side == 1 else fv1, bad if side == 2 else fv2)
        assert _code(M.search_for_triangulation, m, *args, sig2) == fe.ORBFE_ERR_ARG, side
        assert _tri_equal(m, _tri_args(f1, f2, fv1, fv2), sig2) > 0
    # a side-2 feature without a map point in a common node (feature 1, node 7) with an octave outside [0, ORBFE_MAX_LEVELS);
    # sigma2 has an entry for octave 32 all the same
    for octave in (-1, MAX_LEVELS):
        kps2 = f2.kps.copy()
        kps2[1]["octave"] = octave
        args = (f1.kps, f1.desc, f1.flag, fv1, kps2, f2.desc, f2.flag, fv2, S.F12_LINE_Y)
        assert _code(M.search_for_triangulation, m, *args, S.sigma2(33)) == fe.ORBFE_ERR_ARG, octave
        assert _tri_equal(m, _tri_args(f1, f2, fv1, fv2), sig2) > 0
    m.close()


def test_feature_vectors_with_empty_nodes(gpu_required):
    f1, f2, fv1, fv2 = _sparse_pair(seed=5)
    assert len(fv1[0]) > len(f1.desc) and len(fv2[0]) > len(f2.desc)
    for ori in (False, True):
        m = fe.ORBmatcher(0.75, ori)
        f1.flag[:], f2.flag[:] = 1, 1
        for variant in (0, 1):
            assert _bow_equal(m, _bow_args(variant, f1, f2, fv1, fv2)) > 0
        f1.flag[:], f2.flag[:] = 0, 0
        assert _tri_equal(m, _tri_args(f1, f2, fv1, fv2), S.sigma2(8)) > 0
        m.close()


def test_search_by_bow_variant_0_without_valid2(gpu_required):
    f1, f2, E = S.bow_boundary_pair()
    L = M._bind()
    a = np.ascontiguousarray
    fv1, fv2 = [a(x, np.int32) for x in f1.fv()], [a(x, np.int32) for x in f2.fv()]
    a1, a2 = a(f1.kps["angle"], np.float32), a(f2.kps["angle"], np.float32)
    for ori in (False, True):
        m = fe.ORBmatcher(0.75, ori)
        n_o, o_o = O.search_by_bow(0, f1.desc, f1.flag, a1, fv1, f2.desc, f2.flag, a2, fv2, nnratio=0.75, check_orientation=ori)
        out = np.full(len(f2.desc), -9, np.int32)
        nm = C.c_int(-9)
        rc = L.orbfe_search_by_bow(m.handle, 0, len(f1.desc), M._p(f1.desc), M._p(f1.flag), M._p(a1), len(fv1[0]), M._p(fv1[0]),
                                   M._p(fv1[1]), M._p(fv1[2]), len(f2.desc), M._p(f2.desc), None, M._p(a2), len(fv2[0]),
                                   M._p(fv2[0]), M._p(fv2[1]), M._p(fv2[2]), 0.75, int(ori), M._p(out), C.byref(nm))
        assert rc == fe.ORBFE_OK
        assert nm.value == n_o > 0 and np.array_equal(out, o_o), ori
        m.close()


@pytest.mark.parametrize("kind", ["bow", "tri"])
def test_at_most_65535_features_per_side(gpu_required, kind):
    m = fe.ORBmatcher(0.75, True)
    for cap in (65536, 65535):
        f1, f2, E = S.big_pair(kind, cap=cap)
        fv1, fv2 = f1.fv(), f2.fv()
        if kind == "bow":
            for variant in (0, 1):
                args = _bow_args(variant, f1, f2, fv1, fv2)
                if cap == 65536:
                    assert _code(M.search_by_bow, m, *args) == fe.ORBFE_ERR_UNSUPPORTED
                else:
                    assert _bow_equal(m, args) == len(E.applicable())
        else:
            args = _tri_args(f1, f2, fv1, fv2)
            if cap == 65536:
                assert _code(M.search_for_triangulation, m, *args, S.sigma2(8)) == fe.ORBFE_ERR_UNSUPPORTED
            else:
                assert _tri_equal(m, args, S.sigma2(8)) == len(E.applicable())
    m.close()
