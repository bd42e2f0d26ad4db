"""CPU tests of the score entry points (include/orbfe_bow.h orbfe_bow_min_score_device, orbfe_bow_score): every bad argument
is rejected, with a message in orbfe_last_error, before the handle is used (the handles below are zeroed host buffers, never
real handles, and the device pointers are never followed)."""
import ctypes as C

import numpy as np
import pytest

import orb_slam_b200 as fe
from orb_slam_b200 import bow as B

MAX_CAP = 16384   # ORBFE_FV_MAX_CAP


def _fake_handle():
    buf = C.create_string_buffer(4096)
    return buf, C.c_void_p(C.addressof(buf))


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


def _last_error():
    return fe.lib().orbfe_last_error().decode()


def test_bow_min_score_device_rejects_bad_arguments():
    L = B._bind()
    keep, v = _fake_handle()
    d = [C.c_void_p(0x1000 + 0x100 * k) for k in range(8)]   # ids, vals, n, query_row, cov_ptr, cov_row, scores, min_score

    def call(voc=v, nqueries=2, nframes=8, cap=64, ptrs=d):
        return L.orbfe_bow_min_score_device(voc, nqueries, nframes, cap, *ptrs, None)

    assert call(voc=None) == fe.ORBFE_ERR_ARG
    assert call(nqueries=-1) == fe.ORBFE_ERR_ARG
    assert call(nframes=0) == fe.ORBFE_ERR_ARG
    assert call(nframes=-2) == fe.ORBFE_ERR_ARG
    assert call(cap=0) == fe.ORBFE_ERR_ARG
    assert call(cap=-5) == fe.ORBFE_ERR_ARG
    assert "bad arguments" in _last_error()
    for k in range(8):
        ptrs = list(d)
        ptrs[k] = None
        if k == 6:
            continue          # d_scores may be NULL: that call reaches the handle, and is made on a device in the GPU tests
        assert call(ptrs=ptrs) == fe.ORBFE_ERR_ARG, k
        assert "NULL" in _last_error()
    assert call(cap=MAX_CAP + 1) == fe.ORBFE_ERR_UNSUPPORTED
    assert str(MAX_CAP) in _last_error() and "shared memory" in _last_error()
    assert call(nframes=2 ** 31 // 64, cap=64) == fe.ORBFE_ERR_ARG             # nframes * cap = 2^31
    assert "31 bits" in _last_error()
    assert call(nframes=2 ** 31 - 1, cap=MAX_CAP) == fe.ORBFE_ERR_ARG
    assert call(nqueries=0) == fe.ORBFE_OK                                       # nothing to do: the handle is not touched
    assert call(nqueries=0, ptrs=[None] * 8) == fe.ORBFE_OK


def test_bow_score_rejects_bad_arguments():
    L = B._bind()
    keep, v = _fake_handle()
    n = MAX_CAP + 1
    ids, vals = np.arange(n, dtype=np.int32), np.ones(n)
    out = C.c_double(7.0)

    def call(voc=v, n1=4, i1=_p(ids), v1=_p(vals), n2=5, i2=_p(ids), v2=_p(vals), o=C.byref(out)):
        return L.orbfe_bow_score(voc, n1, i1, v1, n2, i2, v2, o)

    assert call(voc=None) == fe.ORBFE_ERR_ARG
    assert call(n1=-1) == fe.ORBFE_ERR_ARG
    assert call(n2=-1) == fe.ORBFE_ERR_ARG
    assert call(o=None) == fe.ORBFE_ERR_ARG
    assert "bad arguments" in _last_error()
    for kw in ("i1", "v1", "i2", "v2"):
        assert call(**{kw: None}) == fe.ORBFE_ERR_ARG, kw
        assert "NULL" in _last_error()
    assert call(n1=MAX_CAP + 1) == fe.ORBFE_ERR_UNSUPPORTED
    assert call(n2=MAX_CAP + 1) == fe.ORBFE_ERR_UNSUPPORTED
    assert str(MAX_CAP + 1) in _last_error() and "shared memory" in _last_error()
    assert out.value == 7.0                                                      # no rejected call wrote the result


def test_python_score_checks_lengths():
    V = B.Vocabulary.__new__(B.Vocabulary)   # no handle: the lengths are checked before the library is called
    V._h = None
    with pytest.raises(ValueError, match="length"):
        V.score([1, 2], [0.5], [1], [1.0])
