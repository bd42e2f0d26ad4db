"""CPU tests of the BowVector entry points (include/orbfe_bow.h orbfe_bow_vector_device, orbfe_bow_transform,
orbfe_kfdb_add_device): bad arguments are rejected before the handle is used (the handles below are zeroed host buffers, never real handles); and the
oracle's BowVector, which the device kernel is tested against, equals DBoW2's own transform() for all four
(weighting, norm) pairs on a vocabulary where the order of every sum shows in the result."""
import ctypes as C
import os

import numpy as np
import pytest

import oracle as O
import orb_slam_b200 as fe
from oracle import ref as R
from orb_slam_b200 import bow as B

import bow_vector_scenes as S

MAX_CAP = 16384   # ORBFE_FV_MAX_CAP


def _fake_handle():
    buf = C.create_string_buffer(4096)
    return buf, C.c_void_p(C.addressof(buf))


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


def test_bow_vector_device_rejects_bad_arguments():
    L = B._bind()
    keep, v = _fake_handle()
    d = [C.c_void_p(0x1000 + 0x100 * k) for k in range(5)]

    def call(voc=v, nframes=2, cap=64, ptrs=d):
        return L.orbfe_bow_vector_device(voc, nframes, ptrs[0], ptrs[1], cap, ptrs[2], ptrs[3], ptrs[4], None)

    assert call(voc=None) == fe.ORBFE_ERR_ARG
    assert call(nframes=-1) == fe.ORBFE_ERR_ARG
    assert call(cap=0) == fe.ORBFE_ERR_ARG
    assert call(cap=-5) == fe.ORBFE_ERR_ARG
    for k in range(5):
        ptrs = list(d)
        ptrs[k] = None
        assert call(ptrs=ptrs) == fe.ORBFE_ERR_ARG, k
    assert call(cap=MAX_CAP + 1) == fe.ORBFE_ERR_UNSUPPORTED
    assert b"" != fe.lib().orbfe_last_error()
    assert call(nframes=0) == fe.ORBFE_OK                 # nothing to do: the handle is not touched


def test_bow_transform_rejects_bad_arguments():
    """orbfe_bow_transform: NULL handle, n < 0 and NULL outputs are ORBFE_ERR_ARG; more descriptors than the kernels sort in
    shared memory is ORBFE_ERR_UNSUPPORTED with the counts and fv_ptr[0] left 0; n = 0 is OK.  None of these touches the
    handle."""
    L = B._bind()
    keep, v = _fake_handle()
    n = MAX_CAP + 1
    desc = np.zeros((n, 32), np.uint8)
    bow_ids, bow_vals = np.zeros(n, np.int32), np.zeros(n, np.float64)
    fv_ids, fv_ptr, fv_feats = np.zeros(n, np.int32), np.full(n + 1, 7, np.int32), np.zeros(n, np.int32)
    nw, nn = C.c_int(7), C.c_int(7)
    outs = [C.byref(nw), _p(bow_ids), _p(bow_vals), C.byref(nn), _p(fv_ids), _p(fv_ptr), _p(fv_feats)]

    def call(voc=v, n=4, desc=_p(desc), outs=outs):
        return L.orbfe_bow_transform(voc, desc, n, 4, *outs)

    assert call(voc=None) == fe.ORBFE_ERR_ARG
    assert call(n=-1) == fe.ORBFE_ERR_ARG
    assert call(desc=None) == fe.ORBFE_ERR_ARG
    for k in range(len(outs)):
        o = list(outs)
        o[k] = None
        assert call(outs=o) == fe.ORBFE_ERR_ARG, k
    nw.value = nn.value = fv_ptr[0] = 7
    assert call(n=MAX_CAP + 1) == fe.ORBFE_ERR_UNSUPPORTED
    assert b"" != fe.lib().orbfe_last_error()
    assert nw.value == 0 and nn.value == 0 and fv_ptr[0] == 0
    nw.value = nn.value = fv_ptr[0] = 7
    assert call(n=0, desc=None) == fe.ORBFE_OK            # nothing to do: the handle is not touched
    assert nw.value == 0 and nn.value == 0 and fv_ptr[0] == 0


def test_kfdb_add_device_rejects_bad_arguments():
    L = B._bind_kfdb()
    keep, h = _fake_handle()
    d = [C.c_void_p(0x1000 + 0x100 * k) for k in range(3)]
    ok_slots, ok_frames = np.array([0, 3, 1], np.int32), np.array([2, 0, 1], np.int32)

    def call(db=h, n=3, slots=ok_slots, frames=ok_frames, cap=64, ptrs=d):
        return L.orbfe_kfdb_add_device(db, n, _p(slots) if slots is not None else None, _p(frames) if frames is not None else None,
                                       cap, ptrs[0], ptrs[1], ptrs[2], None)

    assert call(db=None) == fe.ORBFE_ERR_ARG
    assert call(n=-1) == fe.ORBFE_ERR_ARG
    for cap in (0, -1, MAX_CAP + 1):
        assert call(cap=cap) == fe.ORBFE_ERR_ARG, cap
    assert call(slots=None) == fe.ORBFE_ERR_ARG
    assert call(frames=None) == fe.ORBFE_ERR_ARG
    for k in range(3):
        ptrs = list(d)
        ptrs[k] = None
        assert call(ptrs=ptrs) == fe.ORBFE_ERR_ARG, k
    assert call(slots=np.array([0, -1, 1], np.int32)) == fe.ORBFE_ERR_ARG      # negative slot
    assert call(slots=np.array([0, 3, 0], np.int32)) == fe.ORBFE_ERR_ARG       # repeated slot
    assert call(frames=np.array([2, -1, 1], np.int32)) == fe.ORBFE_ERR_ARG     # negative frame
    assert call(n=0) == fe.ORBFE_OK                                           # nothing to add: the handle is not touched


def test_order_vocabulary_discriminates_summation_order():
    """The sums the tests rely on: on this vocabulary numpy's pairwise sum of a frame's norm terms differs from the
    sequential one, for L1 and L2, and so does the BowVector normalised by it."""
    voc = S.order_vocabulary()
    desc = S.frame_descriptors(voc, 2000, seed=7)
    leaf, _ = O.bow_descend(voc, desc, 0)
    for weighting, norm in S.MODES:
        ids, raw = S.raw_word_values(voc, leaf, weighting)
        assert len(ids) > 100
        (oi, ov), _ = O.bow_transform(voc, desc, 0, weighting, norm)
        pi, pv = S.py_bow_vector(voc, leaf, weighting, norm)
        assert np.array_equal(oi, pi) and np.array_equal(ov.view(np.uint64), pv.view(np.uint64)), (weighting, norm)
        if norm != B.NORM_NONE:
            seq, pair = S.sequential_norm(raw, norm), S.pairwise_norm(raw, norm)
            assert seq != pair, (weighting, norm)
            assert not np.array_equal(pv, np.asarray(raw) / pair)


@pytest.mark.skipif(not (R.available() or os.path.isdir(os.path.join(R.REFERENCE_ROOT, "src"))),
                    reason="oracle/_ref is built from the reference sources, which are absent, and no prebuilt library is present")
@pytest.mark.parametrize("weighting,norm", S.MODES)
def test_oracle_bow_vector_equals_dbow2_on_order_vocabulary(tmp_path, weighting, norm):
    """DBoW2::TemplatedVocabulary::transform itself (loaded from the text format with this weighting and a scoring type that
    asks for this norm) vs the oracle's BowVector, bit for bit."""
    voc = S.order_vocabulary()
    path = str(tmp_path / "voc.txt")
    R.write_vocabulary_text(voc, path, scoring=S.SCORING_OF_NORM[norm], weighting=weighting)
    V = R.RefVocabulary(path)
    desc = S.frame_descriptors(voc, 2000, seed=7)
    for levelsup in (0, 2):
        (bi, bv), _ = V.transform(desc, levelsup)
        (obi, obv), _ = O.bow_transform(voc, desc, levelsup, weighting, norm)
        assert np.array_equal(bi, obi) and np.array_equal(bv.view(np.uint64), obv.view(np.uint64)), levelsup
        assert len(bi) > 100
