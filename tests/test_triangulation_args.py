"""CPU test of the device-resident SearchForTriangulation entry point: bad arguments are rejected with ORBFE_ERR_ARG before the
matcher handle or a device is touched (the handle below is a zeroed host buffer, never a real handle)."""
import ctypes as C

import orb_slam_b200 as fe
from orb_slam_b200 import matching as M

CAP = 64
NLEVELS = 8


def _fake_handle():
    buf = C.create_string_buffer(256)
    return buf, C.c_void_p(C.addressof(buf))


def _ptrs(n):
    """n distinct non-NULL addresses that must never be dereferenced."""
    bufs = [C.create_string_buffer(8) for _ in range(n)]
    return bufs, [C.c_void_p(C.addressof(b)) for b in bufs]


def test_search_for_triangulation_device_rejects_bad_arguments():
    L = M._bind()
    keep, h = _fake_handle()
    # kps, desc, counts, fv_ids, fv_ptr, fv_items, fv_n, has_mp, idx1, idx2, F12, sigma2, match12, nmatches
    bufs, p = _ptrs(14)

    def call(m=h, njobs=4, cap=CAP, nlevels=NLEVELS, args=None):
        a = list(p) if args is None else args
        return L.orbfe_search_for_triangulation_device(m, njobs, a[0], a[1], a[2], cap, a[3], a[4], a[5], a[6], a[7], a[8], a[9],
                                                       a[10], a[11], nlevels, 1, a[12], a[13], None)

    assert call(cap=0) == fe.ORBFE_ERR_ARG
    assert call(cap=65536) == fe.ORBFE_ERR_ARG
    assert call(nlevels=0) == fe.ORBFE_ERR_ARG
    assert call(nlevels=33) == fe.ORBFE_ERR_ARG
    assert call(njobs=-1) == fe.ORBFE_ERR_ARG
    assert call(m=None) == fe.ORBFE_ERR_ARG
    for k in range(14):   # every pointer, the host array sigma2 (k = 11) included
        a = list(p)
        a[k] = None
        assert call(args=a) == fe.ORBFE_ERR_ARG, k
    assert b"" != fe.lib().orbfe_last_error()
    # nothing to do: accepted without reading any pointer
    assert call(njobs=0, args=[None] * 14) == fe.ORBFE_OK
