"""CPU test of the covisibility-graph entries and orbfe_kfdb_set_covisibles_device: bad arguments are rejected with
ORBFE_ERR_ARG before the handle or a device is touched (the handle below is a zeroed host buffer, never a real handle)."""
import ctypes as C

import numpy as np

import orb_slam_b200 as fe
from orb_slam_b200 import bow as B


def _fake_handle():
    buf = C.create_string_buffer(256)
    return buf, C.c_void_p(C.addressof(buf))


def _ptrs(n):
    bufs = [C.create_string_buffer(32) for _ in range(n)]
    return bufs, [C.c_void_p(C.addressof(b)) for b in bufs]


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


def test_create_rejects_bad_arguments():
    L = B._bind_kfdb()
    h = C.c_void_p()
    for args in ((0, 0, 8, 4), (0, 16, 0, 4), (0, 16, 2049, 4), (0, 16, 8, 0), (0, 16, 8, 1025), (-1, 16, 8, 4), (0, 1 << 20, 2048, 4)):
        assert L.orbfe_covis_create(*args, C.byref(h)) == fe.ORBFE_ERR_ARG, args
        assert h.value is None
    assert L.orbfe_covis_create(0, 16, 8, 4, None) == fe.ORBFE_ERR_ARG


def test_entries_reject_bad_arguments_before_the_handle():
    L = B._bind_kfdb()
    keep, h = _fake_handle()
    bufs, p = _ptrs(8)
    slots = np.array([0, 1, 2], np.int32)
    ids = np.array([0, 1, 2], np.int32)
    keys = np.array([5, 6, 7], np.uint64)
    # add
    assert L.orbfe_covis_add(None, 3, _p(slots), _p(ids), _p(keys)) == fe.ORBFE_ERR_ARG
    assert L.orbfe_covis_add(h, -1, _p(slots), _p(ids), _p(keys)) == fe.ORBFE_ERR_ARG
    for k in range(3):
        a = [_p(slots), _p(ids), _p(keys)]
        a[k] = None
        assert L.orbfe_covis_add(h, 3, *a) == fe.ORBFE_ERR_ARG, k
    neg = np.array([0, -1, 2], np.int32)
    assert L.orbfe_covis_add(h, 3, _p(neg), _p(ids), _p(keys)) == fe.ORBFE_ERR_ARG
    assert L.orbfe_covis_add(h, 0, None, None, None) == fe.ORBFE_OK

    # update_connections_device: (g, n, slots, kf_mp, counts, nframes, cap, gp, obs, npoints, nobs, parent, stream)
    def upd(g=h, n=3, sl=slots, nframes=4, cap=16, npoints=10, nobs=20, args=None):
        a = list(p[:4]) if args is None else args
        return L.orbfe_covis_update_connections_device(g, n, None if sl is None else _p(sl), a[0], a[1], nframes, cap, a[2], a[3], npoints,
                                                       nobs, None, None)
    assert upd(g=None) == fe.ORBFE_ERR_ARG
    assert upd(n=-1) == fe.ORBFE_ERR_ARG
    assert upd(nframes=0) == fe.ORBFE_ERR_ARG
    assert upd(cap=0) == fe.ORBFE_ERR_ARG
    assert upd(nframes=65536, cap=32768) == fe.ORBFE_ERR_ARG   # nframes * cap overflows int32
    assert upd(npoints=-1) == fe.ORBFE_ERR_ARG
    assert upd(nobs=-1) == fe.ORBFE_ERR_ARG
    assert upd(sl=None) == fe.ORBFE_ERR_ARG
    for k in range(4):
        a = list(p[:4])
        a[k] = None
        assert upd(args=a) == fe.ORBFE_ERR_ARG, k
    assert upd(sl=np.array([0, 1, 1], np.int32)) == fe.ORBFE_ERR_ARG          # repeated
    assert upd(sl=np.array([0, 4, 1], np.int32)) == fe.ORBFE_ERR_ARG          # >= nframes
    assert upd(sl=np.array([0, -2, 1], np.int32)) == fe.ORBFE_ERR_ARG
    assert b"orbfe_covis_update_connections_device" in fe.lib().orbfe_last_error()
    assert upd(n=0, sl=None, args=[None] * 4) == fe.ORBFE_OK
    # erase / clear / sync
    assert L.orbfe_covis_erase(None, 0) == fe.ORBFE_ERR_ARG
    assert L.orbfe_covis_erase(h, -1) == fe.ORBFE_ERR_ARG
    assert L.orbfe_covis_clear(None) == fe.ORBFE_ERR_ARG
    assert L.orbfe_covis_sync(None) == fe.ORBFE_ERR_ARG

    # lists_device: (g, which, n, slots, nbest, ptr, list, weights, stream)
    def lst(g=h, which=0, n=3, sl=slots, args=None):
        a = list(p[4:6]) if args is None else args
        return L.orbfe_covis_lists_device(g, which, n, None if sl is None else _p(sl), 10, a[0], a[1], None, None)
    assert lst(g=None) == fe.ORBFE_ERR_ARG
    assert lst(which=2) == fe.ORBFE_ERR_ARG
    assert lst(which=-1) == fe.ORBFE_ERR_ARG
    assert lst(n=-1) == fe.ORBFE_ERR_ARG
    assert lst(sl=None) == fe.ORBFE_ERR_ARG
    assert lst(args=[None, p[5]]) == fe.ORBFE_ERR_ARG
    assert lst(args=[p[4], None]) == fe.ORBFE_ERR_ARG
    assert lst(sl=np.array([0, -1, 2], np.int32)) == fe.ORBFE_ERR_ARG
    assert lst(n=0, sl=None, args=[None, None]) == fe.ORBFE_OK


def test_set_covisibles_device_rejects_bad_arguments_before_the_handle():
    L = B._bind_kfdb()
    keep, h = _fake_handle()
    bufs, p = _ptrs(2)
    slots = np.array([0, 1], np.int32)
    assert L.orbfe_kfdb_set_covisibles_device(None, 2, _p(slots), p[0], p[1], None) == fe.ORBFE_ERR_ARG
    assert L.orbfe_kfdb_set_covisibles_device(h, -1, _p(slots), p[0], p[1], None) == fe.ORBFE_ERR_ARG
    assert L.orbfe_kfdb_set_covisibles_device(h, 2, None, p[0], p[1], None) == fe.ORBFE_ERR_ARG
    assert L.orbfe_kfdb_set_covisibles_device(h, 2, _p(slots), None, p[1], None) == fe.ORBFE_ERR_ARG
    assert L.orbfe_kfdb_set_covisibles_device(h, 2, _p(slots), p[0], None, None) == fe.ORBFE_ERR_ARG
    neg = np.array([0, -3], np.int32)
    assert L.orbfe_kfdb_set_covisibles_device(h, 2, _p(neg), p[0], p[1], None) == fe.ORBFE_ERR_ARG
    assert L.orbfe_kfdb_set_covisibles_device(h, 0, None, None, None, None) == fe.ORBFE_OK
