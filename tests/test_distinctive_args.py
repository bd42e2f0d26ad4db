"""CPU test of the device-resident ComputeDistinctiveDescriptors entry point: bad arguments are rejected with ORBFE_ERR_ARG
before the matcher handle or a device is touched (the handle below is a zeroed host buffer, never a real handle)."""
import ctypes as C

import orb_slam_b200 as fe
from orb_slam_b200 import bow as B

CAP = 64
NFRAMES = 3


def _fake_handle():
    buf = C.create_string_buffer(256)
    return buf, C.c_void_p(C.addressof(buf))


def _ptrs(n):
    """n distinct non-NULL, 16-byte aligned addresses that must never be dereferenced."""
    bufs = [C.create_string_buffer(32) for _ in range(n)]
    return bufs, [C.c_void_p((C.addressof(b) + 15) & ~15) for b in bufs]


def test_distinctive_descriptors_device_rejects_bad_arguments():
    L = B._bind()
    keep, h = _fake_handle()
    # desc, counts, group_ptr, obs, best, mp_desc
    bufs, p = _ptrs(6)

    def call(m=h, ngroups=4, nframes=NFRAMES, cap=CAP, nobs=10, args=None):
        a = list(p) if args is None else args
        return L.orbfe_distinctive_descriptors_device(m, ngroups, a[0], a[1], nframes, cap, a[2], a[3], nobs, a[4], a[5], None)

    assert call(m=None) == fe.ORBFE_ERR_ARG
    assert call(ngroups=-1) == fe.ORBFE_ERR_ARG
    assert call(nobs=-1) == fe.ORBFE_ERR_ARG
    assert call(cap=0) == fe.ORBFE_ERR_ARG
    assert call(cap=65536) == fe.ORBFE_ERR_ARG
    assert call(nframes=0) == fe.ORBFE_ERR_ARG
    assert call(nframes=-2) == fe.ORBFE_ERR_ARG
    assert call(nframes=32769, cap=65535) == fe.ORBFE_ERR_ARG   # nframes * cap overflows int32
    assert call(nframes=65536, cap=32768) == fe.ORBFE_ERR_ARG
    for k in range(6):
        a = list(p)
        a[k] = None
        assert call(args=a) == fe.ORBFE_ERR_ARG, k
    # the descriptor rows are read and written with 16-byte accesses
    for k in (0, 5):
        a = list(p)
        a[k] = C.c_void_p(a[k].value + 4)
        assert call(args=a) == fe.ORBFE_ERR_ARG, k
    assert b"orbfe_distinctive_descriptors_device" in fe.lib().orbfe_last_error()
    # nothing to do: accepted without reading any pointer
    assert call(ngroups=0, args=[None] * 6) == fe.ORBFE_OK
    assert call(ngroups=0, nobs=0) == fe.ORBFE_OK
