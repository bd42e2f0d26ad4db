"""CPU tests of the mixed-geometry extract entries (include/orbfe.h orbfe_extract_multi, orbfe_extract_multi_device):
malformed arguments are rejected with ORBFE_ERR_ARG before the handle is used (the handle below is a zeroed host buffer,
never a real handle)."""
import ctypes as C

import numpy as np

import orb_slam_b200 as fe


def _fake_handle():
    buf = C.create_string_buffer(4096)
    return buf, C.c_void_p(C.addressof(buf))


def _groups(*specs):
    """specs: (width, height, stride, batch, imgs pointer)"""
    arr = (fe.OrbfeImageGroup * max(len(specs), 1))()
    for g, (w, h, stride, b, p) in zip(arr, specs):
        g.width, g.height, g.stride, g.frame_stride, g.batch, g.imgs = w, h, stride, stride * max(h, 0), b, p
    return arr


IMG = 0x1000   # never dereferenced: every call below fails its argument checks first


def _calls(h, ngroups, groups, cap=1000):
    """(host form, device form) status of one argument set, with valid output buffers"""
    L = fe.lib()
    kps, desc, n = np.zeros(4, fe.KP_DTYPE), np.zeros((4, 32), np.uint8), np.zeros(64, np.int32)
    host = L.orbfe_extract_multi(h, ngroups, groups, kps.ctypes.data, desc.ctypes.data, cap, n.ctypes.data)
    dev = L.orbfe_extract_multi_device(h, ngroups, groups, 0x2000, 0x3000, 0x4000, None)
    return host, dev


def test_group_count_outside_the_limit_is_rejected():
    keep, h = _fake_handle()
    limit = fe.ORBFE_MULTI_MAX_GROUPS
    ok = [(640, 480, 640, 1, IMG)] * (limit + 1)
    for n in (0, -1, limit + 1):
        assert _calls(h, n, _groups(*ok)) == (fe.ORBFE_ERR_ARG, fe.ORBFE_ERR_ARG), n
    assert b"" != fe.lib().orbfe_last_error()


def test_null_groups_and_null_handle_are_rejected():
    keep, h = _fake_handle()
    assert _calls(h, 1, None) == (fe.ORBFE_ERR_ARG, fe.ORBFE_ERR_ARG)
    assert _calls(None, 1, _groups((640, 480, 640, 1, IMG))) == (fe.ORBFE_ERR_ARG, fe.ORBFE_ERR_ARG)


def test_bad_group_is_rejected_wherever_it_stands():
    keep, h = _fake_handle()
    good = (640, 480, 640, 1, IMG)
    for bad in ((640, 480, 640, 0, IMG), (640, 480, 640, -2, IMG),   # batch <= 0
                (640, 480, 639, 1, IMG), (1281, 720, 1280, 2, IMG),  # stride < width
                (0, 480, 640, 0, IMG), (640, 480, 640, 0, None)):    # an empty group still needs batch >= 1
        for specs in ((bad,), (good, bad), (bad, good, good)):
            assert _calls(h, len(specs), _groups(*specs)) == (fe.ORBFE_ERR_ARG, fe.ORBFE_ERR_ARG), (bad, len(specs))


def test_more_than_65535_frames_across_groups_are_rejected():
    """one grid row per frame: 65536 frames split across groups are ORBFE_ERR_ARG before the handle is used"""
    keep, h = _fake_handle()
    for split in ((65535, 1), (32768, 32768), (1, 1, 65534)):
        groups = _groups(*[(640, 480, 640, b, IMG) for b in split])
        assert _calls(h, len(split), groups) == (fe.ORBFE_ERR_ARG, fe.ORBFE_ERR_ARG), split
        assert b"65536 frames" in fe.lib().orbfe_last_error()


def test_null_outputs_and_negative_cap_are_rejected():
    L = fe.lib()
    keep, h = _fake_handle()
    groups = _groups((640, 480, 640, 2, IMG), (320, 240, 320, 1, IMG))
    kps, desc, n = np.zeros(4, fe.KP_DTYPE), np.zeros((4, 32), np.uint8), np.zeros(3, np.int32)
    K, D, N = kps.ctypes.data, desc.ctypes.data, n.ctypes.data
    for args in ((None, D, 10, N), (K, None, 10, N), (K, D, 10, None), (K, D, -1, N)):
        assert L.orbfe_extract_multi(h, 2, groups, *args) == fe.ORBFE_ERR_ARG, args
    for args in ((None, 0x3000, 0x4000), (0x2000, None, 0x4000), (0x2000, 0x3000, None)):
        assert L.orbfe_extract_multi_device(h, 2, groups, *args, None) == fe.ORBFE_ERR_ARG, args


def test_plan_builds_of_no_handle_is_zero():
    assert fe.lib().orbfe_extractor_plan_builds(None) == 0
