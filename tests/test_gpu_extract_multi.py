"""orbfe_extract_multi / orbfe_extract_multi_device: frames of several image geometries in one call.

Every frame's keypoints (all seven fields, angles bit for bit), descriptors and count must equal what
orbfe_extract_batch_device gives for that frame's geometry on a second handle with the same constructor arguments; one set is
also compared with the oracle.  Groups use non-tight strides: some are read in place, some copied (a stride that is not a
multiple of 16 bytes)."""
import os
import subprocess
import sys

import numpy as np
import pytest

import oracle as O
import orb_slam_b200 as fe
from orb_slam_b200.synth import textured_frame
from multi_domain_scenes import empty_levels

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SPIN = 100_000_000          # torch.cuda._sleep cycles: one bounded spin of roughly 50 ms on an H100

SETS = {
    "1080p_720p_vga": [(1920, 1080, 3), (1280, 720, 1), (640, 480, 2)],
    "landscape_portrait": [(640, 480, 2), (480, 640, 1)],
    "odd_sizes": [(641, 479, 2), (1001, 333, 1)],
    "repeated": [(640, 480, 1), (1280, 720, 2), (640, 480, 3)],
}
SETTINGS = {   # nfeatures, scaleFactor, nlevels, scoreType, fastTh
    "fast_th20_8lv": (1000, 1.2, 8, fe.FAST_SCORE, 20),
    "harris_th20_8lv": (1000, 1.2, 8, fe.HARRIS_SCORE, 20),
    "fast_th5_6lv": (1500, 1.2, 6, fe.FAST_SCORE, 5),
    "harris_th7_4lv": (800, 1.3, 4, fe.HARRIS_SCORE, 7),
}


def _torch():
    import torch
    return torch, torch.device("cuda", 0)


class Group:
    """`b` frames of one geometry in a host buffer with `row_pad` bytes after each row and `frame_pad` after each frame"""

    def __init__(self, w, h, b, seed, row_pad=0, frame_pad=0):
        self.w, self.h, self.b = w, h, b
        self.frames = np.stack([textured_frame(w, h, seed=seed + i) for i in range(b)])
        self.stride = w + row_pad
        self.frame_stride = self.stride * h + frame_pad
        self.buf = np.full(self.frame_stride * b, 77, np.uint8)
        for i in range(b):
            self.buf[i * self.frame_stride:i * self.frame_stride + self.stride * h].reshape(h, self.stride)[:, :w] = self.frames[i]
        self.d = None

    def dev(self):
        if self.d is None:
            torch, dev = _torch()
            self.d = torch.from_numpy(self.buf).to(dev)
        return self.d


# in place (tight), in place (16-byte aligned padding), copied (odd row stride)
PADS = [(0, 0), (16, 32), (3, 5)]


def _groups(spec, seed=0):
    return [Group(w, h, b, seed + 100 * i, *PADS[i % len(PADS)]) for i, (w, h, b) in enumerate(spec)]


def _slots(ex):
    return int(ex.tables()[2].sum())


class Out:
    """device outputs for F frames"""

    def __init__(self, ex, F):
        torch, dev = _torch()
        self.cap, self.F = _slots(ex), F
        self.kps = torch.zeros((F, self.cap, 28), dtype=torch.uint8, device=dev)
        self.desc = torch.zeros((F, self.cap, 32), dtype=torch.uint8, device=dev)
        self.cnt = torch.full((F,), -1, dtype=torch.int32, device=dev)

    def host(self):
        k = self.kps.cpu().numpy().view(fe.KP_DTYPE).reshape(self.F, self.cap)
        return [(k[f, :c], d[:c]) for f, (c, d) in enumerate(zip(self.cnt.cpu().numpy(), self.desc.cpu().numpy()))]


def multi_device(ex, groups, stream=0, out=None):
    out = out or Out(ex, sum(g.b for g in groups))
    ex.extract_multi_device([(g.dev().data_ptr(), g.w, g.h, g.stride, g.frame_stride, g.b) for g in groups],
                            out.kps.data_ptr(), out.desc.data_ptr(), out.cnt.data_ptr(), stream)
    return out


def single_device(ex, g, stream=0):
    out = Out(ex, g.b)
    ex.extract_batch_device(g.dev().data_ptr(), g.w, g.h, g.stride, g.frame_stride, g.b, out.kps.data_ptr(),
                            out.desc.data_ptr(), out.cnt.data_ptr(), stream)
    return out


def reference(params, groups):
    """per frame, orbfe_extract_batch_device on that frame's geometry, on a handle of its own"""
    torch, _ = _torch()
    ref = fe.ORBextractor(*params)
    try:
        res = []
        for g in groups:
            out = single_device(ref, g)
            torch.cuda.synchronize()
            res += out.host()
        return res
    finally:
        ref.close()


def same(got, want, tag):
    assert len(got) == len(want), (tag, len(got), len(want))
    for f, ((gk, gd), (wk, wd)) in enumerate(zip(got, want)):
        assert len(gk) == len(wk), (tag, f, len(gk), len(wk))
        for name in ("x", "y", "size", "response", "octave", "class_id"):
            assert np.array_equal(gk[name], wk[name]), (tag, f, name)
        assert np.array_equal(gk["angle"].view(np.uint32), wk["angle"].view(np.uint32)), (tag, f)
        assert np.array_equal(gd, wd), (tag, f)


@pytest.mark.parametrize("setting", sorted(SETTINGS))
@pytest.mark.parametrize("geoms", sorted(SETS))
def test_multi_equals_single_geometry_entry(gpu_required, geoms, setting):
    torch, _ = _torch()
    params = SETTINGS[setting]
    groups = _groups(SETS[geoms], seed=len(geoms))
    ex = fe.ORBextractor(*params)
    try:
        out = multi_device(ex, groups)
        torch.cuda.synchronize()
        got = out.host()
        assert ex.last_launches() == params[2] + 4
    finally:
        ex.close()
    want = reference(params, groups)
    assert sum(len(k) for k, _ in want) > 0
    same(got, want, (geoms, setting))


def test_multi_with_empty_cell_grid_levels(gpu_required):
    torch, _ = _torch()
    params = (200, 1.2, 8, fe.FAST_SCORE, 20)
    spec = [(640, 480, 1), (1001, 333, 2), (480, 640, 1)]
    assert empty_levels(params, 1001, 333) and empty_levels(params, 480, 640) and not empty_levels(params, 640, 480)
    groups = _groups(spec, seed=5)
    ex = fe.ORBextractor(*params)
    try:
        out = multi_device(ex, groups)
        torch.cuda.synchronize()
        got = out.host()
    finally:
        ex.close()
    same(got, reference(params, groups), "empty levels")


def test_multi_equals_the_oracle(gpu_required):
    torch, _ = _torch()
    groups = _groups([(1280, 720, 1), (640, 480, 2), (480, 640, 1)], seed=11)
    ex = fe.ORBextractor(1000, 1.2, 8, fe.FAST_SCORE, 20)
    try:
        got = multi_device(ex, groups)
        torch.cuda.synchronize()
        got = got.host()
    finally:
        ex.close()
    want = []
    for g in groups:
        for img in g.frames:
            rc, k, d, _ = O.extract(O.make_params(1000, 1.2, 8, 1, 20), img)
            assert rc == 0
            want.append((k, d))
    same(got, want, "oracle")


@pytest.mark.parametrize("ngroups", [1, 2, 3])
def test_launch_count_does_not_grow_with_groups(gpu_required, ngroups):
    torch, _ = _torch()
    groups = _groups([(640, 480, 1), (1280, 720, 2), (480, 640, 1)][:ngroups])
    for nl in (8, 5):
        ex = fe.ORBextractor(1000, 1.2, nl, fe.FAST_SCORE, 20)
        try:
            multi_device(ex, groups)
            torch.cuda.synchronize()
            assert ex.last_launches() == nl + 4, (ngroups, nl)
        finally:
            ex.close()


def test_alternating_calls_do_not_replan(gpu_required):
    torch, _ = _torch()
    params = SETTINGS["fast_th20_8lv"]
    single = Group(1280, 720, 2, seed=40)
    big = _groups([(640, 480, 2), (1280, 720, 1), (480, 640, 2)], seed=50)
    small = _groups([(640, 480, 1), (1280, 720, 1), (480, 640, 2)], seed=60)   # the same geometries, fewer frames
    want_single = reference(params, [single])
    want_big, want_small = reference(params, big), reference(params, small)
    ex = fe.ORBextractor(*params)
    try:
        assert ex.plan_builds() == 0
        for r in range(4):
            s = single_device(ex, single)
            m = multi_device(ex, big if r % 2 == 0 else small)
            torch.cuda.synchronize()
            same(s.host(), want_single, ("single", r))
            same(m.host(), want_big if r % 2 == 0 else want_small, ("multi", r))
            assert ex.plan_builds() == 2, r
    finally:
        ex.close()


def test_multi_and_single_on_two_streams_run_in_call_order(gpu_required):
    """A spin on stream A, then a multi call on A, a single call on B and a second multi call on B (other frames, the same
    geometries): every result is the one of running the three calls in call order."""
    torch, dev = _torch()
    params = SETTINGS["fast_th20_8lv"]
    A, Bs = torch.cuda.Stream(device=dev), torch.cuda.Stream(device=dev)
    g1 = _groups([(640, 480, 1), (1280, 720, 2)], seed=70)
    g2 = _groups([(640, 480, 1), (1280, 720, 2)], seed=80)
    single = Group(480, 640, 2, seed=90)
    want1, want2, want_s = reference(params, g1), reference(params, g2), reference(params, [single])
    ex = fe.ORBextractor(*params)
    try:
        for g in g1 + g2 + [single]:
            g.dev()
        o1, o2 = Out(ex, 3), Out(ex, 3)
        multi_device(ex, g1, out=o1)          # load every kernel once, without a spin in front
        single_device(ex, single)
        torch.cuda.synchronize()
        with torch.cuda.stream(A):
            torch.cuda._sleep(SPIN)
        multi_device(ex, g1, A.cuda_stream, out=o1)
        s = single_device(ex, single, Bs.cuda_stream)
        multi_device(ex, g2, Bs.cuda_stream, out=o2)
        torch.cuda.synchronize()
        same(o1.host(), want1, "first multi")
        same(s.host(), want_s, "single")
        same(o2.host(), want2, "second multi")
    finally:
        ex.close()


_PDL_SCRIPT = r"""
import sys, numpy as np
sys.path.insert(0, sys.argv[1]); sys.path.insert(0, sys.argv[1] + "/tests")
import torch, orb_slam_b200 as fe
import test_gpu_extract_multi as T
ex = fe.ORBextractor(*T.SETTINGS[sys.argv[3]])
out = T.multi_device(ex, T._groups(T.SETS["1080p_720p_vga"], seed=3))
torch.cuda.synchronize()
res = out.host()
np.savez(sys.argv[2], cnt=np.array([len(k) for k, _ in res]), kps=np.concatenate([k for k, _ in res]),
         desc=np.concatenate([d for _, d in res]))
"""


@pytest.mark.parametrize("setting", ["fast_th20_8lv", "harris_th20_8lv"])
def test_pdl_off_gives_the_same_results(gpu_required, tmp_path, setting):
    torch, _ = _torch()
    env = dict(os.environ, ORBFE_PDL="0")
    path = str(tmp_path / "pdl0.npz")
    subprocess.run([sys.executable, "-c", _PDL_SCRIPT, ROOT, path, setting], env=env, check=True, timeout=600)
    ex = fe.ORBextractor(*SETTINGS[setting])
    try:
        out = multi_device(ex, _groups(SETS["1080p_720p_vga"], seed=3))
        torch.cuda.synchronize()
        got = out.host()
    finally:
        ex.close()
    z = np.load(path)
    splits = np.cumsum(z["cnt"])[:-1]
    same(got, list(zip(np.split(z["kps"], splits), np.split(z["desc"], splits))), ("pdl off", setting))


@pytest.mark.parametrize("cap_extra", [0, 37])
def test_host_form_equals_device_form(gpu_required, cap_extra):
    torch, _ = _torch()
    params = SETTINGS["harris_th20_8lv"]
    groups = _groups(SETS["repeated"], seed=21)
    ex = fe.ORBextractor(*params)
    try:
        dev = multi_device(ex, groups)
        torch.cuda.synchronize()
        want = dev.host()
        cap = _slots(ex) + cap_extra
        got = ex.extract_multi([g.frames for g in groups], cap=cap)
        assert ex.plan_builds() == 1
    finally:
        ex.close()
    same(got, want, "host form")


def test_empty_groups_yield_no_keypoints(gpu_required):
    torch, _ = _torch()
    params = SETTINGS["fast_th20_8lv"]
    g = _groups([(640, 480, 2), (1280, 720, 1)], seed=31)
    ex = fe.ORBextractor(*params)
    try:
        out = Out(ex, 6)
        ex.extract_multi_device([(g[0].dev().data_ptr(), 640, 480, g[0].stride, g[0].frame_stride, 2), (0, 640, 480, 640, 640 * 480, 1),
                                 (g[1].dev().data_ptr(), 1280, 720, g[1].stride, g[1].frame_stride, 1),
                                 (g[1].dev().data_ptr(), 0, 0, 0, 0, 2)],
                                out.kps.data_ptr(), out.desc.data_ptr(), out.cnt.data_ptr())
        torch.cuda.synchronize()
        got = out.host()
        host = ex.extract_multi([g[0].frames, None, g[1].frames, np.zeros((0, 0), np.uint8)])
    finally:
        ex.close()
    want = reference(params, g)
    same([got[0], got[1], got[3]], want, "device form")
    same([host[0], host[1], host[3]], want, "host form")
    assert (out.cnt.cpu().numpy()[[2, 4, 5]] == 0).all()
    assert len(host) == 5 and len(host[2][0]) == 0 and len(host[4][0]) == 0
    for f in (2, 4, 5):
        assert len(got[f][0]) == 0, f


def test_unsupported_group_is_named_and_nothing_runs(gpu_required):
    torch, _ = _torch()
    g = _groups([(640, 480, 1)], seed=1)[0]
    ex = fe.ORBextractor(1000, 1.2, 8, fe.FAST_SCORE, 20)
    try:
        out = Out(ex, 2)
        with pytest.raises(fe.OrbfeError) as e:
            ex.extract_multi_device([(g.dev().data_ptr(), 640, 480, 640, 640 * 480, 1), (g.dev().data_ptr(), 40, 30, 640, 640 * 480, 1)],
                                    out.kps.data_ptr(), out.desc.data_ptr(), out.cnt.data_ptr())
        assert e.value.code == fe.ORBFE_ERR_UNSUPPORTED and "group 1" in str(e.value)
        torch.cuda.synchronize()
        assert (out.cnt.cpu().numpy() == -1).all()
        assert ex.plan_builds() == 0 and ex.last_launches() == 0
    finally:
        ex.close()
