"""CPU test of orbfe_covis_keyframe_culling_device: bad arguments are rejected before the handle or a device is touched (the
handle is a zeroed host buffer, never a real handle), each with its status."""
import ctypes as C

import orb_slam_b200 as fe
from orb_slam_b200 import bow as B


def test_keyframe_culling_device_rejects_bad_arguments_before_the_handle():
    L = B._bind_kfdb()
    buf = C.create_string_buffer(256)
    h = C.c_void_p(C.addressof(buf))
    keep = [C.create_string_buffer(64) for _ in range(16)]
    p = [C.c_void_p(C.addressof(b)) for b in keep]
    odd = C.c_void_p(C.addressof(keep[15]) + 2)
    ne = (C.c_int32 * 2)(0, 1)
    bad_ne = (C.c_int32 * 1)(-1)

    def call(g=h, cur=0, kf_mp=p[0], counts=p[1], kps=p[2], nframes=4, cap=16, point_bad=p[3], ref_slot=p[4], npoints=10, n_ne=0,
             ne_slots=None, obs_cap=8, nobs=p[5], vs=p[6], vd=p[7], ncand=p[8], nm=None, nr=None, bp=p[9], nbad=p[10], scratch=p[11]):
        return L.orbfe_covis_keyframe_culling_device(g, cur, kf_mp, counts, kps, nframes, cap, point_bad, ref_slot, npoints, n_ne, ne_slots,
                                                     obs_cap, nobs, vs, vd, ncand, nm, nr, bp, nbad, scratch, None)

    ARG = fe.ORBFE_ERR_ARG
    cases = [
        dict(g=None), dict(npoints=-1), dict(nframes=0), dict(cap=0), dict(obs_cap=-1), dict(n_ne=-1),
        dict(nframes=1 << 16, cap=1 << 15),                       # nframes * cap >= 2^31
        dict(kf_mp=None), dict(counts=None), dict(kps=None), dict(nobs=None), dict(vs=None), dict(vd=None), dict(ncand=None),
        dict(nbad=None), dict(scratch=None), dict(point_bad=None), dict(ref_slot=None), dict(bp=None),
        dict(n_ne=1, ne_slots=None),                               # mbNotErase slots missing
        dict(scratch=odd),                                         # not 4-byte aligned
        dict(cur=0), dict(cur=-1), dict(cur=5),                    # no live slot in a zeroed handle
    ]
    for kw in cases:
        assert call(**kw) == ARG, kw
        assert b"orbfe_covis_keyframe_culling_device" in fe.lib().orbfe_last_error(), kw
    assert call(cap=8193) == fe.ORBFE_ERR_UNSUPPORTED   # ORBFE_COVIS_OBS_MAX_CAP + 1
    assert call(n_ne=1, ne_slots=bad_ne) == ARG
    assert call(n_ne=2, ne_slots=ne) == ARG              # the current slot is still not live
    # npoints = 0 needs no per-point arrays: the current slot is what is refused
    assert call(npoints=0, point_bad=None, ref_slot=None, bp=None) == ARG
    assert b"current slot" in fe.lib().orbfe_last_error()
