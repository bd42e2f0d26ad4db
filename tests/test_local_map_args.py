"""CPU test of orbfe_covis_local_map_device: bad arguments are rejected before the handle or a device is touched (the handle
is a zeroed host buffer, never a real handle), each with its status."""
import ctypes as C

import orb_slam_b200 as fe
from orb_slam_b200 import bow as B


def test_local_map_device_rejects_bad_arguments_before_the_handle():
    L = B._bind_kfdb()
    buf = C.create_string_buffer(256)
    h = C.c_void_p(C.addressof(buf))
    keep = [C.create_string_buffer(64) for _ in range(12)]
    p = [C.c_void_p(C.addressof(b)) for b in keep]
    odd = C.c_void_p(C.addressof(keep[11]) + 2)

    def call(g=h, nf=4, frame=p[0], point_bad=p[1], npoints=10, kf_mp=p[2], counts=p[3], nframes=4, cap=16, lk=p[4], nlk=p[5], ref=p[6],
             lp=p[7], nlp=p[8], scratch=p[9]):
        return L.orbfe_covis_local_map_device(g, nf, frame, point_bad, npoints, kf_mp, counts, nframes, cap, lk, nlk, ref, lp, nlp, scratch,
                                              None)

    ARG = fe.ORBFE_ERR_ARG
    cases = [
        dict(g=None), dict(nf=-1), dict(npoints=-1), dict(nframes=0), dict(cap=0),
        dict(nframes=1 << 16, cap=1 << 15),                       # nframes * cap >= 2^31
        dict(frame=None), dict(point_bad=None), dict(kf_mp=None), dict(counts=None), dict(lk=None), dict(nlk=None), dict(ref=None),
        dict(lp=None), dict(nlp=None), dict(scratch=None),
        dict(scratch=odd),                                         # not 4-byte aligned
    ]
    for kw in cases:
        assert call(**kw) == ARG, kw
        assert b"orbfe_covis_local_map_device" in fe.lib().orbfe_last_error(), kw
    assert call(cap=8193) == fe.ORBFE_ERR_UNSUPPORTED   # ORBFE_COVIS_OBS_MAX_CAP + 1
    assert b"cap 8193" in fe.lib().orbfe_last_error()
