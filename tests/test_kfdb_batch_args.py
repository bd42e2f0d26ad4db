"""CPU tests of the batched keyframe-database entries (include/orbfe_bow.h orbfe_kfdb_create_batched,
orbfe_kfdb_detect_batch_device): malformed arguments are rejected with ORBFE_ERR_ARG before the handle is used (the handles
below are zeroed host buffers, never real handles)."""
import ctypes as C

import orb_slam_b200 as fe
from orb_slam_b200 import bow as B

from test_kfdb_args import _fake_handle


def test_create_batched_rejects_bad_arguments():
    L = B._bind_kfdb()
    keep, v = _fake_handle()
    out = C.c_void_p()
    for K, P, Q in ((4, 10, 0), (4, 10, -1), (4, 10, 1025), (0, 10, 1), ((1 << 24) + 1, 10, 1), (4, 0, 1), (4, 1 << 31, 1)):
        assert L.orbfe_kfdb_create_batched(v, K, P, Q, C.byref(out)) == fe.ORBFE_ERR_ARG, (K, P, Q)
        assert not out.value
    assert L.orbfe_kfdb_create_batched(None, 4, 10, 1, C.byref(out)) == fe.ORBFE_ERR_ARG
    assert L.orbfe_kfdb_create_batched(v, 4, 10, 1, None) == fe.ORBFE_ERR_ARG
    assert b"" != fe.lib().orbfe_last_error()


def test_detect_batch_device_rejects_bad_arguments():
    L = B._bind_kfdb()
    keep, h = _fake_handle()
    vp = C.c_void_p
    d = [vp(0x1000 + 0x100 * i) for i in range(8)]

    def call(db=h, mode=1, nqueries=2, qcap=3, ids=d[0], vals=d[1], ptr=d[2], conn=d[3], ms=d[4], cap=4, cand=d[5], ncand=d[6]):
        return L.orbfe_kfdb_detect_batch_device(db, mode, nqueries, qcap, ids, vals, ptr, conn, ms, cap, cand, ncand, None, None, None)

    for kw in (dict(mode=2), dict(mode=-1), dict(nqueries=0), dict(nqueries=-3), dict(qcap=-1), dict(qcap=65536), dict(cap=-1),
               dict(cap=4, cand=None), dict(ncand=None), dict(ids=None), dict(vals=None), dict(mode=0, ptr=None), dict(mode=0, ms=None),
               dict(db=None)):
        assert call(**kw) == fe.ORBFE_ERR_ARG, kw
