"""CPU tests of the keyframe-database entry points (include/orbfe_bow.h orbfe_kfdb_*): malformed arguments are rejected with
ORBFE_ERR_ARG before the handle is used (the handle below is a zeroed host buffer, never a real handle)."""
import ctypes as C

import numpy as np

import orb_slam_b200 as fe
from orb_slam_b200 import bow as B


def _fake_handle():
    buf = C.create_string_buffer(4096)
    return buf, C.c_void_p(C.addressof(buf))


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


def test_create_rejects_bad_arguments():
    L = B._bind_kfdb()
    keep, v = _fake_handle()
    out = C.c_void_p()
    for K, P in ((0, 10), (-1, 10), ((1 << 24) + 1, 10), (4, 0), (4, 1 << 31)):
        assert L.orbfe_kfdb_create(v, K, P, C.byref(out)) == fe.ORBFE_ERR_ARG, (K, P)
        assert not out.value
    assert L.orbfe_kfdb_create(None, 4, 10, C.byref(out)) == fe.ORBFE_ERR_ARG
    assert L.orbfe_kfdb_create(v, 4, 10, None) == fe.ORBFE_ERR_ARG


def test_add_rejects_bad_arguments():
    L = B._bind_kfdb()
    keep, h = _fake_handle()
    ok_ids, vals = np.array([1, 4, 9], np.int32), np.ones(3)
    for slot, ids in ((-1, ok_ids), (0, np.array([1, 9, 4], np.int32)), (0, np.array([1, 4, 4], np.int32)),
                      (0, np.array([-2, 4, 9], np.int32))):                          # slot < 0, unsorted, repeated, negative id
        assert L.orbfe_kfdb_add(h, slot, 3, _p(ids), _p(vals)) == fe.ORBFE_ERR_ARG, (slot, ids)
    assert L.orbfe_kfdb_add(h, 0, -1, _p(ok_ids), _p(vals)) == fe.ORBFE_ERR_ARG
    assert L.orbfe_kfdb_add(h, 0, 3, None, _p(vals)) == fe.ORBFE_ERR_ARG
    assert L.orbfe_kfdb_add(h, 0, 3, _p(ok_ids), None) == fe.ORBFE_ERR_ARG
    assert L.orbfe_kfdb_add(None, 0, 3, _p(ok_ids), _p(vals)) == fe.ORBFE_ERR_ARG
    assert L.orbfe_kfdb_erase(h, -1) == fe.ORBFE_ERR_ARG
    assert L.orbfe_kfdb_erase(None, 0) == fe.ORBFE_ERR_ARG
    assert L.orbfe_kfdb_clear(None) == fe.ORBFE_ERR_ARG
    assert b"" != fe.lib().orbfe_last_error()


def test_set_covisibles_rejects_bad_arguments():
    L = B._bind_kfdb()
    keep, h = _fake_handle()
    slots = np.array([0, 1], np.int32)
    lists = np.arange(12, dtype=np.int32)
    for ptr in ((0, 11, 12), (1, 2, 3), (0, 3, 2)):                                   # 11 covisibles, ptr[0] != 0, decreasing
        assert L.orbfe_kfdb_set_covisibles(h, 2, _p(slots), _p(np.array(ptr, np.int32)), _p(lists)) == fe.ORBFE_ERR_ARG, ptr
    ptr = np.array([0, 2, 4], np.int32)
    assert L.orbfe_kfdb_set_covisibles(h, 2, _p(np.array([0, -1], np.int32)), _p(ptr), _p(lists)) == fe.ORBFE_ERR_ARG
    assert L.orbfe_kfdb_set_covisibles(h, 2, _p(slots), _p(ptr), _p(np.array([0, -3, 1, 2], np.int32))) == fe.ORBFE_ERR_ARG
    assert L.orbfe_kfdb_set_covisibles(h, 2, _p(slots), _p(ptr), None) == fe.ORBFE_ERR_ARG
    assert L.orbfe_kfdb_set_covisibles(h, -1, _p(slots), _p(ptr), _p(lists)) == fe.ORBFE_ERR_ARG
    assert L.orbfe_kfdb_set_covisibles(h, 2, None, _p(ptr), _p(lists)) == fe.ORBFE_ERR_ARG
    assert L.orbfe_kfdb_set_covisibles(None, 2, _p(slots), _p(ptr), _p(lists)) == fe.ORBFE_ERR_ARG


def test_detect_rejects_bad_arguments():
    L = B._bind_kfdb()
    keep, h = _fake_handle()
    q, qv = np.array([1, 4, 9], np.int32), np.ones(3)
    conn, out = np.zeros(4, np.int32), np.zeros(64, np.int32)
    n, words, score = C.c_int(0), np.zeros(64, np.int32), np.zeros(64, np.float32)

    def call(db=h, mode=1, nq=3, ids=q, nconn=0, cap=16, ncand=True, cand=out):
        return L.orbfe_kfdb_detect(db, mode, nq, _p(ids) if ids is not None else None, _p(qv), nconn, _p(conn), 0.0, cap,
                                   _p(cand) if cand is not None else None, C.byref(n) if ncand else None, _p(words), _p(score))

    assert call(mode=2) == fe.ORBFE_ERR_ARG
    assert call(mode=-1) == fe.ORBFE_ERR_ARG
    assert call(cap=-1) == fe.ORBFE_ERR_ARG
    assert call(cap=4, cand=None) == fe.ORBFE_ERR_ARG
    assert call(nq=-1) == fe.ORBFE_ERR_ARG
    assert call(nq=65536) == fe.ORBFE_ERR_ARG
    assert call(nconn=-1) == fe.ORBFE_ERR_ARG
    assert call(ids=np.array([4, 1, 9], np.int32)) == fe.ORBFE_ERR_ARG
    assert call(ids=np.array([-1, 1, 9], np.int32)) == fe.ORBFE_ERR_ARG
    assert call(ids=None) == fe.ORBFE_ERR_ARG
    assert call(ncand=False) == fe.ORBFE_ERR_ARG
    assert call(db=None) == fe.ORBFE_ERR_ARG
    vp = C.c_void_p
    dev = [vp(0x1000)] * 8
    assert L.orbfe_kfdb_detect_device(h, 3, 3, dev[0], dev[1], 0, dev[2], 0.0, 4, dev[3], dev[4], None, None, None) == fe.ORBFE_ERR_ARG
    assert L.orbfe_kfdb_detect_device(h, 1, 3, dev[0], dev[1], 0, dev[2], 0.0, -2, dev[3], dev[4], None, None, None) == fe.ORBFE_ERR_ARG
    assert L.orbfe_kfdb_detect_device(h, 1, 3, None, dev[1], 0, dev[2], 0.0, 4, dev[3], dev[4], None, None, None) == fe.ORBFE_ERR_ARG
    assert L.orbfe_kfdb_detect_device(h, 0, 3, dev[0], dev[1], 2, None, 0.0, 4, dev[3], dev[4], None, None, None) == fe.ORBFE_ERR_ARG
    assert L.orbfe_kfdb_detect_device(h, 1, 3, dev[0], dev[1], 0, None, 0.0, 4, dev[3], None, None, None, None) == fe.ORBFE_ERR_ARG
