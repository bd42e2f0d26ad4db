"""CPU tests of the device-resident SearchByBoW entry points: bad arguments are rejected with ORBFE_ERR_ARG before the
matcher / vocabulary handle or a device is touched (the handle below is a zeroed host buffer, never a real handle)."""
import ctypes as C

import orb_slam_b200 as fe
from orb_slam_b200 import bow as B
from orb_slam_b200 import matching as M

CAP = 64


def _fake_handle():
    buf = C.create_string_buffer(256)
    return buf, C.c_void_p(C.addressof(buf))


def _ptrs(n):
    """n distinct non-NULL addresses that must never be dereferenced."""
    bufs = [C.create_string_buffer(8) for _ in range(n)]
    return bufs, [C.c_void_p(C.addressof(b)) for b in bufs]


def test_search_by_bow_device_rejects_bad_arguments():
    L = M._bind()
    keep, h = _fake_handle()
    bufs, p = _ptrs(12)
    kps, desc, cnt, ids, ptr, items, nfv, valid, i1, i2, out, nm = p

    def call(m=h, variant=0, njobs=4, cap=CAP, args=None):
        a = list(p) if args is None else args
        return L.orbfe_search_by_bow_device(m, variant, njobs, a[0], a[1], a[2], cap, a[3], a[4], a[5], a[6], a[7], a[8], a[9],
                                            0.75, 1, a[10], a[11], None)

    assert call(variant=2) == fe.ORBFE_ERR_ARG
    assert call(variant=-1) == fe.ORBFE_ERR_ARG
    assert call(cap=0) == fe.ORBFE_ERR_ARG
    assert call(cap=65536) == fe.ORBFE_ERR_ARG
    assert call(njobs=-1) == fe.ORBFE_ERR_ARG
    assert call(m=None) == fe.ORBFE_ERR_ARG
    for k in range(12):
        a = list(p)
        a[k] = None
        assert call(args=a) == fe.ORBFE_ERR_ARG, k
    assert b"" != fe.lib().orbfe_last_error()
    # nothing to do: accepted without reading any pointer
    assert call(njobs=0, args=[None] * 12) == fe.ORBFE_OK


def test_feature_vector_device_rejects_bad_arguments():
    L = B._bind()
    keep, h = _fake_handle()
    bufs, p = _ptrs(7)

    def call(m=h, nframes=3, cap=CAP, args=None):
        a = list(p) if args is None else args
        return L.orbfe_feature_vector_device(m, nframes, a[0], a[1], a[2], cap, a[3], a[4], a[5], a[6], None)

    assert call(nframes=-1) == fe.ORBFE_ERR_ARG
    assert call(cap=0) == fe.ORBFE_ERR_ARG
    assert call(m=None) == fe.ORBFE_ERR_ARG
    for k in range(7):
        a = list(p)
        a[k] = None
        assert call(args=a) == fe.ORBFE_ERR_ARG, k
    # a frame capacity whose sort keys do not fit in shared memory
    assert call(cap=16385) == fe.ORBFE_ERR_UNSUPPORTED
    assert call(nframes=0, args=[None] * 7) == fe.ORBFE_OK
