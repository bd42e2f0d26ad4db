"""CPU tests of the camera-table matcher entries (include/orbfe_match.h orbfe_search_by_projection_cams_device,
orbfe_search_for_initialization_cams_device, orbfe_guided_search_cams_device): malformed arguments are rejected with
ORBFE_ERR_ARG before the handle is used (the handle below is a zeroed host buffer, never a real handle)."""
import ctypes as C
import math

import orb_slam_b200 as fe
from orb_slam_b200 import matching as M

GOOD = (0.0, 0.0, 1280.0, 720.0, 900.0, 900.0, 640.0, 360.0)
D = 0x1000   # never dereferenced: every call below fails its argument checks first


def _fake_handle():
    buf = C.create_string_buffer(4096)
    return buf, C.c_void_p(C.addressof(buf))


def _calls(h, ncams, cams, frame_cam=D, n=2, cap=1000, qcap=64, nlevels=8, rule=1, window=100, ptr=D):
    """status of the three entries for one argument set"""
    L = M._bind()
    sbp = L.orbfe_search_by_projection_cams_device(h, n, ptr, D, D, cap, D, D, D, D, D, ncams, cams, frame_cam, 1.2, nlevels, 7.0,
                                                   1, D, D, None)
    init = L.orbfe_search_for_initialization_cams_device(h, n, ptr, D, D, cap, D, D, D, ncams, cams, frame_cam, window, 0.9, 1, D,
                                                         D, None)
    guided = L.orbfe_guided_search_cams_device(h, n, ptr, D, D, cap, D, D, D, D, D, D, D, D, D, D, qcap, ncams, cams, frame_cam,
                                               rule, 0.8, 100, 1, D, D, None)
    return sbp, init, guided


ARG3 = (fe.ORBFE_ERR_ARG,) * 3


def test_camera_count_outside_the_limit_is_rejected():
    keep, h = _fake_handle()
    limit = fe.ORBFE_MULTI_MAX_GROUPS
    cams = M.cameras([GOOD] * (limit + 1))
    for n in (0, -1, limit + 1, 1 << 30):
        assert _calls(h, n, cams) == ARG3, n
    assert b"ncams" in fe.lib().orbfe_last_error()


def test_null_table_and_null_frame_cameras_are_rejected():
    keep, h = _fake_handle()
    assert _calls(h, 1, None) == ARG3
    assert _calls(h, 1, M.cameras([GOOD]), frame_cam=None) == ARG3


def test_bad_bounds_are_rejected_for_any_camera():
    keep, h = _fake_handle()
    nan, inf = math.nan, math.inf
    bad = [(0, 0, 0, 720), (10, 0, 5, 720), (0, 0, 1280, 0), (0, 5, 1280, -5), (nan, 0, 1280, 720), (0, 0, nan, 720),
           (0, nan, 1280, 720), (0, 0, 1280, nan), (-inf, 0, -inf, 720), (inf, 0, inf, 720)]
    for b in bad:
        cam = tuple(b) + GOOD[4:]
        for table in ([cam], [GOOD, cam], [GOOD] * 7 + [cam]):
            assert _calls(h, len(table), M.cameras(table)) == ARG3, (b, len(table))
            assert b"camera %d" % (len(table) - 1) in fe.lib().orbfe_last_error()


def test_the_single_geometry_checks_still_apply():
    """the checks the single-geometry entries make: null handle, negative pair count, cap, level count, query capacity,
    rule, window and NULL device arrays"""
    keep, h = _fake_handle()
    cams = M.cameras([GOOD, GOOD])
    assert _calls(None, 2, cams) == ARG3
    assert _calls(h, 2, cams, n=-1) == ARG3
    assert _calls(h, 2, cams, cap=0) == ARG3
    assert _calls(h, 2, cams, ptr=None) == ARG3
    L = M._bind()
    assert L.orbfe_search_by_projection_cams_device(h, 2, D, D, D, 65536, D, D, D, D, D, 2, cams, D, 1.2, 8, 7.0, 1, D, D,
                                                    None) == fe.ORBFE_ERR_ARG
    for nl in (0, 33):
        assert L.orbfe_search_by_projection_cams_device(h, 2, D, D, D, 1000, D, D, D, D, D, 2, cams, D, 1.2, nl, 7.0, 1, D, D,
                                                        None) == fe.ORBFE_ERR_ARG, nl
    assert L.orbfe_search_for_initialization_cams_device(h, 2, D, D, D, 1000, D, D, D, 2, cams, D, -1, 0.9, 1, D, D,
                                                         None) == fe.ORBFE_ERR_ARG
    assert L.orbfe_search_for_initialization_cams_device(h, 2, D, D, D, 65535, D, D, D, 2, cams, D, 100, 0.9, 1, D, D,
                                                         None) == fe.ORBFE_ERR_ARG
    for qcap, rule in ((0, 1), (65536, 1), (64, -1), (64, 3)):
        assert L.orbfe_guided_search_cams_device(h, 2, D, D, D, 1000, D, D, D, D, D, D, D, D, D, D, qcap, 2, cams, D, rule, 0.8,
                                                 100, 1, D, D, None) == fe.ORBFE_ERR_ARG, (qcap, rule)
    # check_orientation needs the query angles
    assert L.orbfe_guided_search_cams_device(h, 2, D, D, D, 1000, D, D, D, D, D, D, D, None, D, D, 64, 2, cams, D, 1, 0.8, 100, 1,
                                             D, D, None) == fe.ORBFE_ERR_ARG


def test_no_pairs_with_a_valid_table_is_a_no_op():
    keep, h = _fake_handle()
    assert _calls(h, 2, M.cameras([GOOD, GOOD]), n=0) == (fe.ORBFE_OK,) * 3
