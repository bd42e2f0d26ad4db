"""CPU test of orbfe_covis_observations_device: bad arguments are rejected before the handle or a device is touched (the
handle is a zeroed host buffer, never a real handle), each with its status."""
import ctypes as C

import orb_slam_b200 as fe
from orb_slam_b200 import bow as B


def test_observations_device_rejects_bad_arguments_before_the_handle():
    L = B._bind_kfdb()
    buf = C.create_string_buffer(256)
    h = C.c_void_p(C.addressof(buf))
    keep = [C.create_string_buffer(64) for _ in range(8)]
    p = [C.c_void_p(C.addressof(b)) for b in keep]
    odd = C.c_void_p(C.addressof(keep[7]) + 2)

    # (g, n, points, npoints, kf_mp, counts, nframes, cap, ref_slot, obs_cap, ptr, obs, nobs, ref_obs, scratch, stream)
    def call(g=h, n=3, points=p[0], npoints=10, kf_mp=p[1], counts=p[2], nframes=4, cap=16, ref_slot=None, obs_cap=8, ptr=p[3],
             obs=p[4], nobs=p[5], ref_obs=None, scratch=p[6]):
        return L.orbfe_covis_observations_device(g, n, points, npoints, kf_mp, counts, nframes, cap, ref_slot, obs_cap, ptr, obs, nobs,
                                                 ref_obs, scratch, None)

    ARG = fe.ORBFE_ERR_ARG
    cases = [
        dict(g=None), dict(n=-1), dict(npoints=-1), dict(n=11), dict(nframes=0), dict(cap=0), dict(obs_cap=-1),
        dict(nframes=1 << 16, cap=1 << 15),                       # nframes * cap >= 2^31
        dict(points=None), dict(kf_mp=None), dict(counts=None), dict(ptr=None), dict(nobs=None), dict(scratch=None),
        dict(obs=None),                                            # obs_cap > 0
        dict(ref_slot=p[7]), dict(ref_obs=p[7]),                   # one without the other
        dict(scratch=odd),                                         # not 4-byte aligned
    ]
    for kw in cases:
        assert call(**kw) == ARG, kw
        assert b"orbfe_covis_observations_device" in fe.lib().orbfe_last_error(), kw
    assert call(cap=8193) == fe.ORBFE_ERR_UNSUPPORTED   # ORBFE_COVIS_OBS_MAX_CAP + 1
