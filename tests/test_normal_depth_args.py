"""CPU test of both MapPoint::UpdateNormalAndDepth entry points: bad arguments are rejected with ORBFE_ERR_ARG before the
matcher handle or a device is touched (the handle below is a zeroed host buffer, never a real handle)."""
import ctypes as C

import numpy as np

import orb_slam_b200 as fe
from orb_slam_b200 import bow as B

CAP = 64
NFRAMES = 3


def _fake_handle():
    buf = C.create_string_buffer(256)
    return buf, C.c_void_p(C.addressof(buf))


def _ptrs(n):
    """n distinct non-NULL addresses that must never be dereferenced."""
    bufs = [C.create_string_buffer(32) for _ in range(n)]
    return bufs, [C.c_void_p(C.addressof(b)) for b in bufs]


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


def test_normal_and_depth_device_rejects_bad_arguments():
    L = B._bind()
    keep, h = _fake_handle()
    # kps, counts, centers, group_ptr, obs, world, ref_obs, normal, min_dist, max_dist
    bufs, p = _ptrs(10)
    sf = np.ones(32, np.float32)

    def call(m=h, npoints=4, nframes=NFRAMES, cap=CAP, nobs=10, nlevels=8, table=sf, args=None):
        a = list(p) if args is None else args
        return L.orbfe_normal_and_depth_device(m, npoints, a[0], a[1], nframes, cap, a[2], a[3], a[4], nobs, a[5], a[6], 1.2, nlevels,
                                               None if table is None else _p(table), a[7], a[8], a[9], None)

    assert call(m=None) == fe.ORBFE_ERR_ARG
    assert call(npoints=-1) == fe.ORBFE_ERR_ARG
    assert call(nobs=-1) == fe.ORBFE_ERR_ARG
    assert call(cap=0) == fe.ORBFE_ERR_ARG
    assert call(cap=65536) == fe.ORBFE_ERR_ARG
    assert call(nframes=0) == fe.ORBFE_ERR_ARG
    assert call(nframes=-2) == fe.ORBFE_ERR_ARG
    assert call(nframes=32769, cap=65535) == fe.ORBFE_ERR_ARG   # nframes * cap overflows int32
    assert call(nlevels=0) == fe.ORBFE_ERR_ARG
    assert call(nlevels=33) == fe.ORBFE_ERR_ARG
    assert call(table=None) == fe.ORBFE_ERR_ARG
    for k in range(10):
        a = list(p)
        a[k] = None
        assert call(args=a) == fe.ORBFE_ERR_ARG, k
    assert b"orbfe_normal_and_depth_device" in fe.lib().orbfe_last_error()
    # nothing to do: accepted without reading any pointer
    assert call(npoints=0, args=[None] * 10, table=None) == fe.ORBFE_OK
    assert call(npoints=0, nobs=0) == fe.ORBFE_OK


def test_normal_and_depth_host_rejects_bad_arguments():
    L = B._bind()
    keep, h = _fake_handle()
    n = 3
    world = np.zeros((n, 3), np.float32)
    refc = np.zeros((n, 3), np.float32)
    octs = np.array([0, 7, 3], np.int32)
    gp = np.array([0, 2, 2, 5], np.int32)
    obs = np.zeros((5, 3), np.float32)
    sf = np.ones(8, np.float32)
    outn, outa, outb = np.zeros((n, 3), np.float32), np.zeros(n, np.float32), np.zeros(n, np.float32)

    def call(m=h, npoints=n, nlevels=8, **kw):
        a = dict(world=world, refc=refc, octs=octs, gp=gp, obs=obs, sf=sf, outn=outn, outa=outa, outb=outb)
        a.update(kw)
        q = {k: (None if v is None else _p(v)) for k, v in a.items()}
        return L.orbfe_normal_and_depth(m, npoints, q["world"], q["refc"], q["octs"], q["gp"], q["obs"], 1.2, nlevels, q["sf"], q["outn"],
                                        q["outa"], q["outb"])

    assert call(m=None) == fe.ORBFE_ERR_ARG
    assert call(npoints=-1) == fe.ORBFE_ERR_ARG
    assert call(nlevels=0) == fe.ORBFE_ERR_ARG
    assert call(nlevels=33) == fe.ORBFE_ERR_ARG
    for k in ("world", "refc", "octs", "gp", "obs", "sf", "outn", "outa", "outb"):
        assert call(**{k: None}) == fe.ORBFE_ERR_ARG, k
    assert call(gp=np.array([1, 2, 2, 5], np.int32)) == fe.ORBFE_ERR_ARG          # group_ptr[0] != 0
    assert call(gp=np.array([0, 2, 1, 5], np.int32)) == fe.ORBFE_ERR_ARG          # decreasing
    assert call(gp=np.array([0, 0, 0, -1], np.int32)) == fe.ORBFE_ERR_ARG         # negative total
    for bad in (-1, 8, 1 << 30):                                                 # octave of a non-empty point outside [0, 8)
        o = octs.copy()
        o[2] = bad
        assert call(octs=o) == fe.ORBFE_ERR_ARG, bad
    assert b"reference octave" in fe.lib().orbfe_last_error()
    o = octs.copy()
    o[2] = 7
    assert call(octs=o, nlevels=7) == fe.ORBFE_ERR_ARG
    # nothing to do: accepted without reading any pointer
    assert L.orbfe_normal_and_depth(h, 0, None, None, None, None, None, 1.2, 8, None, None, None, None) == fe.ORBFE_OK
    # the rejected calls returned before writing
    assert not outn.any() and not outa.any() and not outb.any()
