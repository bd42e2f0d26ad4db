"""orbfe_extract_multi / orbfe_extract_multi_device at their limits, bit for bit.

The domain scenes of extract_domain_scenes.py and orient_domain_scenes.py as one group among others, at every position;
eight groups of distinct geometries up to the 8 x 32 level table and at scale factors 2.0 and 3.0; tile-less groups
(no FAST tile, no cell) at every position and a handle whose every group is tile-less; the level-select kernel past 48 KB
in a multi plan, in a fresh process whose first plan is a multi plan, and refusals that name the group whose footprint
is too large; the capacity rule over sequences of calls on one handle; every ingest layout in one call; output slots past
each frame's count and the host form's capacity error; a 64-frame group beside others and 65535 frames in one call; and
the frame store of a two-camera call fed to the projection matcher.

Every frame is compared field by field (angles as float32 bits) with its descriptors: domain-scene frames with the
oracle, other frames with the single-geometry entry on a handle of their own or with the oracle."""
import functools
import os
import subprocess
import sys

import numpy as np
import pytest

import oracle as O
import orb_slam_b200 as fe
import extract_domain_scenes as ES
import multi_domain_scenes as S
import orient_domain_scenes as OS
from orb_slam_b200.synth import textured_frame
from test_gpu_extract_domain import _assert_all_kept, _compare, _layout, _level_select_smem, _noise, mixed_frames
from test_gpu_extract_multi import Group, Out, _slots, _torch, multi_device, reference, same

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


class Frames(Group):
    """the given frames [B, H, W] as a group: byte `off` into its device buffer, rows `stride` apart, frames
    `frame_stride` apart, padding 0xA5"""

    def __init__(self, frames, stride=None, frame_stride=None, off=0):
        self.b, self.h, self.w = frames.shape
        self.frames = frames
        self.stride = stride or self.w
        self.frame_stride = frame_stride or self.stride * self.h
        self.off = off
        self.buf = _layout(frames, off, self.stride, self.frame_stride)
        self.d = None

    def dev(self):
        if self.d is None:
            torch, dev = _torch()
            self.d = torch.from_numpy(self.buf).to(dev)[self.off:]
        return self.d


class Empty:
    """a group without images: `b` frames without keypoints"""

    def __init__(self, b):
        self.w = self.h = 0
        self.b = b


class Filled(Out):
    """device outputs for F frames with every byte `fill` and every count -7 (at least one slot per frame)"""

    def __init__(self, ex, F, fill=0xEE):
        torch, dev = _torch()
        self.cap, self.F = max(_slots(ex), 1), F
        self.kps = torch.full((F, self.cap, 28), fill, dtype=torch.uint8, device=dev)
        self.desc = torch.full((F, self.cap, 32), fill, dtype=torch.uint8, device=dev)
        self.cnt = torch.full((F,), -7, dtype=torch.int32, device=dev)


def multi(ex, groups, out=None):
    """multi_device, also with Empty groups among the groups"""
    if not any(isinstance(g, Empty) for g in groups):
        return multi_device(ex, groups, out=out)
    out = out or Out(ex, sum(g.b for g in groups))
    ex.extract_multi_device([(0, 0, 0, 0, 0, g.b) if isinstance(g, Empty) else
                             (g.dev().data_ptr(), g.w, g.h, g.stride, g.frame_stride, g.b) for g in groups],
                            out.kps.data_ptr(), out.desc.data_ptr(), out.cnt.data_ptr())
    return out


def run(params, groups, out=None):
    """one multi call on a new handle: (frames, launches)"""
    torch, _ = _torch()
    ex = fe.ORBextractor(*params)
    try:
        o = multi(ex, groups, out)
        torch.cuda.synchronize()
        return o.host(), ex.last_launches()
    finally:
        ex.close()


def want_of(params, groups):
    """per frame the single-geometry entry's result; Empty groups give empty frames"""
    real = [g for g in groups if not isinstance(g, Empty)]
    res = iter(reference(params, real))
    out = []
    for g in groups:
        for _ in range(g.b):
            out.append((np.zeros(0, fe.KP_DTYPE), np.zeros((0, 32), np.uint8)) if isinstance(g, Empty) else next(res))
    return out


def oracle(params, frames):
    nf, sf, nl, score, th = params
    out = []
    for img in frames:
        rc, k, d, _ = O.extract(O.make_params(nf, sf, nl, score, th), img)
        assert rc == 0
        out.append((k, d))
    return out


def split(got, groups):
    """the call's frames, group by group"""
    res, f = [], 0
    for g in groups:
        res.append(got[f:f + g.b])
        f += g.b
    return res


def partners(seed):
    (W1, H1), (W2, H2) = S.PARTNERS
    return [Group(W1, H1, 1, seed), Group(W2, H2, 2, seed + 50, 16, 32)]


def run_placed(params, scene_groups, pos, seed):
    """the scene's groups at `pos` among the partners; the partners' frames equal the single-geometry entry.  Returns the
    frames of each scene group."""
    ps = partners(seed)
    groups = S.placed(scene_groups, ps, pos)
    got, launches = run(params, groups)
    assert launches == params[2] + 4
    per = split(got, groups)
    want = reference(params, ps)
    same(per[groups.index(ps[0])] + per[groups.index(ps[1])], want, ("partners", pos))
    return [per[groups.index(g)] for g in scene_groups]


# ---------------------------------------------------------------------------------------------------------------------
# 1. domain scenes as one group among others
# ---------------------------------------------------------------------------------------------------------------------
def _threshold_sets(th, score):
    scenes = ES.threshold_scenes(th)
    sparse = ("count", "two_tone_th", "two_tone_th1")
    dense = [n for n in sorted(scenes) if n not in sparse]
    return [((ES.COUNT_NF, 1.2, ES.COUNT_NL, score, th), np.stack([scenes[n] for n in sparse])),
            ((800, 1.2, 3, score, th), np.stack([scenes[n] for n in dense]))]


@pytest.mark.parametrize("pos", S.POSITIONS)
@pytest.mark.parametrize("th,score", [(t, fe.FAST_SCORE) for t in (0, 7, 8, 254)] + [(t, fe.HARRIS_SCORE) for t in (0, 254)])
def test_threshold_scenes_among_groups(gpu_required, th, score, pos):
    for params, frames in _threshold_sets(th, score):
        got, = run_placed(params, [Frames(frames)], pos, seed=th)
        same(got, oracle(params, frames), (th, score, pos, params))


@pytest.mark.parametrize("pos", S.POSITIONS)
@pytest.mark.parametrize("W,H,nl", ES.SEAM_GEOMETRIES)
def test_seam_scene_among_groups(gpu_required, W, H, nl, pos):
    img, pairs = ES.seam_scene(W, H, nl)
    _, p, dump = _compare(img, ES.SEAM_NF, nl, ES.SEAM_TH)
    params = (ES.SEAM_NF, 1.2, nl, fe.FAST_SCORE, ES.SEAM_TH)
    got, = run_placed(params, [Frames(img[None])], pos, seed=W)
    same(got, oracle(params, [img]), (W, H, pos))
    _assert_all_kept(got[0][0], p, dump, W, H)


@pytest.mark.parametrize("pos", S.POSITIONS)
@pytest.mark.parametrize("nlevels", [1, 8])
def test_orient_scenes_among_groups(gpu_required, nlevels, pos):
    """the four interior scenes as one 352 x 272 group and the four border scenes (widths 384-387) as a group each"""
    sc = OS.scenes()
    inner = [s["img"] for s in sc if (s["W"], s["H"]) == (OS.IW, OS.IH)]
    border = [s["img"] for s in sc if (s["W"], s["H"]) != (OS.IW, OS.IH)]
    assert len(inner) == 4 and len(border) == 4
    groups = [Frames(np.stack(inner))] + [Frames(b[None]) for b in border]
    params = (OS.nfeatures(nlevels), 1.2, nlevels, fe.FAST_SCORE, OS.FAST_TH)
    got = run_placed(params, groups, pos, seed=nlevels)
    same(sum(got, []), oracle(params, inner + border), (nlevels, pos))


# ---------------------------------------------------------------------------------------------------------------------
# 2. eight groups
# ---------------------------------------------------------------------------------------------------------------------
def _eight(seed):
    return [Group(W, H, B, seed + 10 * i, *[(0, 0), (16, 32), (3, 5)][i % 3]) for i, ((W, H), B) in enumerate(zip(S.EIGHT, S.EIGHT_BATCH))]


@pytest.mark.parametrize("score", [fe.FAST_SCORE, fe.HARRIS_SCORE])
@pytest.mark.parametrize("setting", sorted(S.EIGHT_SETTINGS))
def test_eight_groups(gpu_required, setting, score):
    nl, sf = S.EIGHT_SETTINGS[setting]
    params = (S.EIGHT_NF, sf, nl, score, 20)
    groups = _eight(seed=nl)
    got, launches = run(params, groups)
    assert launches == nl + 4
    want = reference(params, groups)
    assert all(len(k) > 0 for k, _ in want)
    same(got, want, (setting, score))


def test_eight_groups_equal_the_oracle(gpu_required):
    params = (S.EIGHT_NF, 1.2, 8, fe.FAST_SCORE, 20)
    groups = _eight(seed=3)
    got, _ = run(params, groups)
    same(got, oracle(params, [f for g in groups for f in g.frames]), "oracle")


# ---------------------------------------------------------------------------------------------------------------------
# 3. tile-less groups
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", sorted(S.TILELESS_CALLS))
def test_tileless_group(gpu_required, name):
    """200 x 1200 at nf 100 over 8 levels has no FAST tile and no cell: its frames count 0, every other frame equals the
    single-geometry entry, wherever the group stands"""
    params = S.TILELESS_PARAMS
    groups = [Group(W, H, B, 7 * i) for i, (W, H, B) in enumerate(S.TILELESS_CALLS[name])]
    got, launches = run(params, groups)
    assert launches == params[2] + 4
    for g, frames in zip(groups, split(got, groups)):
        if (g.w, g.h) == S.TILELESS:
            assert all(len(k) == 0 for k, _ in frames), name
    want = reference(params, groups)
    assert sum(len(k) > 0 for k, _ in want) > 0
    same(got, want, name)


def test_nfeatures_zero_every_group_tileless(gpu_required):
    torch, _ = _torch()
    groups = _eight(seed=5)[:4]
    ex = fe.ORBextractor(0, 1.2, 8, fe.FAST_SCORE, 20)
    try:
        out = multi(ex, groups, Filled(ex, sum(g.b for g in groups)))
        torch.cuda.synchronize()
        assert (out.cnt.cpu().numpy() == 0).all()
        assert (out.kps.cpu().numpy() == 0xEE).all() and (out.desc.cpu().numpy() == 0xEE).all()
        assert ex.last_launches() == 8 + 4
    finally:
        ex.close()


# ---------------------------------------------------------------------------------------------------------------------
# 4. level-select shared memory
# ---------------------------------------------------------------------------------------------------------------------
def _noise_groups(spec, seed):
    return [Frames(np.stack([_noise(W, H, seed + 7 * i + f) for f in range(B)])) for i, (W, H, B) in enumerate(spec)]


@pytest.mark.parametrize("key", sorted(S.SMEM_SETS))
def test_level_select_past_48k(gpu_required, key):
    params, spec = S.SMEM_SETS[key]
    nf, sf, nl, score, _ = params
    assert max(_level_select_smem(nf, nl, W, H, score == fe.HARRIS_SCORE, sf) for W, H, _ in spec) == S.Plan(params, spec).smem()[0] > 48 * 1024
    groups = _noise_groups(spec, seed=nf)
    got, _ = run(params, groups)
    same(got, oracle(params, [f for g in groups for f in g.frames]), key)


_SMEM_SCRIPT = r"""
import sys, numpy as np
sys.path.insert(0, sys.argv[1]); sys.path.insert(0, sys.argv[1] + "/tests")
import torch, orb_slam_b200 as fe
import multi_domain_scenes as S
import test_gpu_multi_domain as T
params, spec = S.SMEM_SETS[sys.argv[3]]
(p2, (W, H)) = S.SMEM_SMALLER[sys.argv[3]]
groups = T._noise_groups(spec, seed=params[0])
ex = fe.ORBextractor(*params)
first = T.multi(ex, groups)                      # the first plan this process builds: a multi plan past 48 KB
torch.cuda.synchronize()
other = fe.ORBextractor(*p2)                     # a single-geometry plan needing less, still past 48 KB
k, d = other(T._noise(W, H, 5))
assert len(k) == p2[0]
second = T.multi(ex, groups)
torch.cuda.synchronize()
res = first.host() + second.host()
np.savez(sys.argv[2], cnt=np.array([len(k) for k, _ in res]), kps=np.concatenate([k for k, _ in res]),
         desc=np.concatenate([d for _, d in res]))
"""


@pytest.mark.parametrize("key", sorted(S.SMEM_SETS))
def test_level_select_attribute_in_a_fresh_process(gpu_required, tmp_path, key):
    """The kernel attribute is per process and only grows: a single-geometry plan built after a larger multi plan does
    not lower it, and the multi call still runs and equals the oracle."""
    path = str(tmp_path / "smem.npz")
    subprocess.run([sys.executable, "-c", _SMEM_SCRIPT, ROOT, path, key], check=True, timeout=600)
    params, spec = S.SMEM_SETS[key]
    want = oracle(params, [f for g in _noise_groups(spec, seed=params[0]) for f in g.frames])
    z = np.load(path)
    got = list(zip(np.split(z["kps"], np.cumsum(z["cnt"])[:-1]), np.split(z["desc"], np.cumsum(z["cnt"])[:-1])))
    same(got[:len(want)], want, (key, "first"))
    same(got[len(want):], want, (key, "second"))


@functools.lru_cache(maxsize=None)
def _refusal_want(nf, score, W, H):
    return oracle((nf, 1.2, 1, score, 10), [_noise(W, H, W + H)])[0]


@pytest.mark.parametrize("order", ["runs_first", "refused_first"])
@pytest.mark.parametrize("key", sorted(S.REFUSAL_PAIRS))
def test_level_select_refusal_names_the_group(gpu_required, key, order):
    """nf where one geometry's level-select footprint passes 200 KB and the other's does not: ORBFE_ERR_UNSUPPORTED
    naming the refused group, nothing launched, no plan built; the handle's previous multi call reruns without a rebuild
    and is unchanged; at nf - 1 the pair runs and equals the oracle."""
    torch, _ = _torch()
    score, nf, a, b = S.REFUSAL_PAIRS[key]
    ga, gb = Frames(_noise(*a, a[0] + a[1])[None]), Frames(_noise(*b, b[0] + b[1])[None])
    pair = [ga, gb] if order == "runs_first" else [gb, ga]
    named = pair.index(gb)
    ex = fe.ORBextractor(nf, 1.2, 1, score, 10)
    try:
        prev = multi(ex, [ga])
        torch.cuda.synchronize()
        prev = prev.host()
        builds = ex.plan_builds()
        out = Out(ex, 2)
        with pytest.raises(fe.OrbfeError) as e:
            multi(ex, pair, out)
        msg = str(e.value)
        assert e.value.code == fe.ORBFE_ERR_UNSUPPORTED and ("group %d" % named) in msg and "level-select" in msg, msg
        torch.cuda.synchronize()
        assert (out.cnt.cpu().numpy() == -1).all() and ex.plan_builds() == builds
        again = multi(ex, [ga])
        torch.cuda.synchronize()
        assert ex.plan_builds() == builds
        same(again.host(), prev, (key, order, "rerun"))
    finally:
        ex.close()
    same(prev, reference((nf, 1.2, 1, score, 10), [ga]), (key, "previous"))
    got, _ = run((nf - 1, 1.2, 1, score, 10), pair)
    same(got, [_refusal_want(nf - 1, score, g.w, g.h) for g in pair], (key, order, "nf - 1"))


# ---------------------------------------------------------------------------------------------------------------------
# 5. capacity and re-planning on one handle
# ---------------------------------------------------------------------------------------------------------------------
class Buffer(Group):
    """a caller's device buffer for up to `cap` tight frames of one geometry, rewritten before each call"""

    def __init__(self, W, H, cap):
        torch, dev = _torch()
        self.w, self.h, self.stride, self.frame_stride = W, H, W, W * H
        self.d = torch.zeros(cap * W * H, dtype=torch.uint8, device=dev)

    def load(self, B, seed):
        torch, _ = _torch()
        self.b = B
        self.frames = np.stack([textured_frame(self.w, self.h, seed=seed + f) for f in range(B)])
        self.d.fill_(0)
        self.d[:B * self.w * self.h].copy_(torch.from_numpy(self.frames.reshape(-1)))
        return self


def test_capacity_and_replanning(gpu_required):
    """CAP_SEQUENCE on one handle with each group's caller buffer reused and rewritten between calls (a level 0 left on a
    stale buffer gives wrong keypoints, not a read of freed memory): plan_builds after every call as the rule says;
    then the same geometries in another order rebuild, an inserted empty group does not, and an in-place call on the
    first order's buffers after that rebuild."""
    torch, _ = _torch()
    params = (1000, 1.2, 8, fe.FAST_SCORE, 20)
    bufs = [Buffer(W, H, c) for (W, H), c in zip(S.CAP_GEOMS, S.CAP_MAX)]
    rule = S.capacity([S.spec_of(S.CAP_GEOMS, b) for b in S.CAP_SEQUENCE])
    assert [sum(r for r, _ in rule[:i + 1]) for i in range(len(rule))] == S.CAP_BUILDS
    ex = fe.ORBextractor(*params)
    try:
        for step, batch in enumerate(S.CAP_SEQUENCE):
            groups = [bufs[i].load(B, 100 * step + 10 * i) for i, B in enumerate(batch)]
            out = multi(ex, groups)
            torch.cuda.synchronize()
            assert ex.plan_builds() == S.CAP_BUILDS[step], step
            same(out.host(), reference(params, groups), ("step", step))
        n = S.CAP_BUILDS[-1]
        for tag, order, builds in (("reordered", [1, 0, 2], n + 1), ("empty inserted", [1, None, 0, 2], n + 1),
                                   ("first order", [0, 1, 2], n + 2)):
            groups = [Empty(2) if i is None else bufs[i].load(1 + (i == 2), 900 + 10 * (i or 0) + builds) for i in order]
            out = multi(ex, groups)
            torch.cuda.synchronize()
            assert ex.plan_builds() == builds, tag
            same(out.host(), want_of(params, groups), tag)
    finally:
        ex.close()


# ---------------------------------------------------------------------------------------------------------------------
# 6. ingest per group in one call
# ---------------------------------------------------------------------------------------------------------------------
def _ingest_groups():
    """(W, H, off, stride, frame_stride) per group: in place tight, in place pitched (frame stride past stride * H), the
    2-D copy at base offsets 1, 8 and 15 and with stride W + 1, frame by frame; 640 x 480 both in place and copied"""
    specs = [(640, 480, 0, 640, 640 * 480), (480, 640, 0, 544, 544 * 640 + 4096), (640, 480, 1, 640, 640 * 480),
             (752, 480, 8, 752, 752 * 480), (480, 640, 15, 480, 480 * 640), (752, 480, 0, 753, 753 * 480),
             (640, 480, 8, 641, 641 * 480 + 3)]
    return [Frames(np.stack([textured_frame(W, H, seed=40 + 5 * i + f) for f in range(2)]), stride, fs, off)
            for i, (W, H, off, stride, fs) in enumerate(specs)]


def test_ingest_layouts_in_one_call(gpu_required, monkeypatch):
    params = (1000, 1.2, 8, fe.FAST_SCORE, 20)
    groups = _ingest_groups()
    want = reference(params, groups)
    got, _ = run(params, groups)
    same(got, want, "layouts")
    monkeypatch.setenv("ORBFE_INGEST_COPY", "1")
    got, _ = run(params, groups)
    same(got, want, "ORBFE_INGEST_COPY=1")


def test_host_form_from_noncontiguous_views(gpu_required):
    """row views of a wider array (stride > W), every other frame of a batch (frame stride doubled), a column-strided
    view (copied contiguous by the binding)"""
    params = (1000, 1.2, 8, fe.FAST_SCORE, 20)
    wide = np.stack([textured_frame(700, 500, seed=70 + f) for f in range(2)])
    every = np.stack([textured_frame(480, 640, seed=80 + f) for f in range(4)])
    cols = textured_frame(1504, 480, seed=90)
    views = [wide[:, 7:487, 11:651], every[::2], cols[:, ::2]]
    assert views[0].strides[1] == 700 and views[1].strides[0] == 2 * 480 * 640 and views[2].strides[1] == 2
    ex = fe.ORBextractor(*params)
    try:
        got = ex.extract_multi(views)
    finally:
        ex.close()
    groups = [Frames(np.ascontiguousarray(v if v.ndim == 3 else v[None])) for v in views]
    same(got, reference(params, groups), "host views")


# ---------------------------------------------------------------------------------------------------------------------
# 7. output placement
# ---------------------------------------------------------------------------------------------------------------------
def test_slots_past_each_count_keep_the_sentinel(gpu_required):
    torch, _ = _torch()
    params = (1000, 1.2, 8, fe.FAST_SCORE, 20)
    groups = [Empty(2), Group(640, 480, 2, 11), Empty(1), Group(1280, 720, 1, 12), Empty(1)]
    ex = fe.ORBextractor(*params)
    try:
        out = multi(ex, groups, Filled(ex, 7))
        torch.cuda.synchronize()
        kps, desc, cnt = out.kps.cpu().numpy(), out.desc.cpu().numpy(), out.cnt.cpu().numpy()
        got = out.host()
    finally:
        ex.close()
    want = want_of(params, groups)
    same(got, want, "placement")
    assert list(cnt) == [len(k) for k, _ in want] and cnt[[0, 1, 4, 6]].tolist() == [0, 0, 0, 0]
    for f, c in enumerate(cnt):
        assert (kps[f, c:] == 0xEE).all() and (desc[f, c:] == 0xEE).all(), f


@pytest.mark.parametrize("cap", [0, 1, 700])
def test_host_form_below_the_counts(gpu_required, cap):
    """cap below some frame's count: ORBFE_ERR_CAPACITY, every n_out the true count, each frame's first cap entries
    equal the device form's"""
    params = (1000, 1.2, 8, fe.FAST_SCORE, 20)
    groups = [Group(640, 480, 2, 21), Empty(1), Group(1280, 720, 1, 22)]
    want = want_of(params, groups)
    assert max(len(k) for k, _ in want) > cap
    arr = (fe.OrbfeImageGroup * 3)()
    for a, g in zip(arr, groups):
        a.batch = g.b
        if not isinstance(g, Empty):
            a.width, a.height, a.stride, a.frame_stride, a.imgs = g.w, g.h, g.stride, g.frame_stride, g.buf.ctypes.data
    F = 4
    kps = np.zeros((F, max(cap, 1)), fe.KP_DTYPE)
    desc = np.zeros((F, max(cap, 1), 32), np.uint8)
    n_out = np.full(F, -3, np.int32)
    ex = fe.ORBextractor(*params)
    try:
        rc = fe.lib().orbfe_extract_multi(ex.handle, 3, arr, kps.ctypes.data if cap else None,
                                          desc.ctypes.data if cap else None, cap, n_out.ctypes.data)
    finally:
        ex.close()
    assert rc == fe.ORBFE_ERR_CAPACITY
    assert n_out.tolist() == [len(k) for k, _ in want]
    same([(kps[f, :min(cap, n)], desc[f, :min(cap, n)]) for f, n in enumerate(n_out)],
         [(k[:cap], d[:cap]) for k, d in want], ("cap", cap))


# ---------------------------------------------------------------------------------------------------------------------
# 8. batch sizes
# ---------------------------------------------------------------------------------------------------------------------
def test_batch_of_64_beside_other_groups(gpu_required):
    params = (1000, 1.2, 8, fe.FAST_SCORE, 20)
    mix = Frames(mixed_frames(640, 480, 64))
    others = [Group(1920, 1080, 1, 31), Group(480, 640, 5, 32, 16, 32)]
    groups = [others[0], mix, others[1]]
    got, _ = run(params, groups)
    per = split(got, groups)
    same(per[1], oracle(params, mix.frames), "64 mixed")
    same(per[0] + per[2], reference(params, others), "others")


def test_65535_frames_in_one_call(gpu_required):
    """The grid-row limit: 32768 + 32767 frames, a few distinct frames tiled through each buffer.  Each distinct frame
    equals the oracle, and every copy equals it byte for byte in all its slots.  The handle, the input buffers and the
    outputs take about 716 MB of device memory (measured on an H100 80GB HBM3)."""
    torch, dev = _torch()
    params = S.LIMIT_PARAMS
    groups, distinct = [], []
    for i, (W, H, B) in enumerate(S.LIMIT_GROUPS):
        frames = np.stack([textured_frame(W, H, seed=300 + 10 * i + k) for k in range(S.LIMIT_DISTINCT)])
        distinct.append(frames)
        reps = -(-B // S.LIMIT_DISTINCT)
        g = Frames(frames)
        g.b, g.d = B, torch.from_numpy(frames).to(dev).repeat(reps, 1, 1)[:B].contiguous().view(-1)
        groups.append(g)
    F = sum(g.b for g in groups)
    assert F == S.MAX_FRAMES
    torch.cuda.synchronize()
    free0 = torch.cuda.mem_get_info()[0]
    ex = fe.ORBextractor(*params)
    try:
        out = multi(ex, groups)
        torch.cuda.synchronize()
        used = free0 - torch.cuda.mem_get_info()[0]
        print("65535 frames: %.1f MB of device memory for the handle and the outputs" % (used / 2 ** 20))
        kps, desc, cnt = out.kps.cpu().numpy(), out.desc.cpu().numpy(), out.cnt.cpu().numpy()
    finally:
        ex.close()
    f0 = 0
    for g, frames in zip(groups, distinct):
        want = oracle(params, frames)
        assert sum(len(k) for k, _ in want) > 0
        for k in range(S.LIMIT_DISTINCT):
            f = f0 + k
            same([(kps[f].reshape(-1).view(fe.KP_DTYPE)[:cnt[f]], desc[f, :cnt[f]])], [want[k]], ("distinct", g.w, k))
            idx = np.arange(f, f0 + g.b, S.LIMIT_DISTINCT)
            assert (cnt[idx] == cnt[f]).all() and (kps[idx] == kps[f]).all() and (desc[idx] == desc[f]).all(), (g.w, k)
        f0 += g.b


# ---------------------------------------------------------------------------------------------------------------------
# 9. the frame store feeds the matchers unchanged
# ---------------------------------------------------------------------------------------------------------------------
def test_two_camera_frame_store_feeds_the_projection_matcher(gpu_required):
    """1280 x 720 x 3 and 640 x 480 x 3 in one call; orbfe_search_by_projection_device pairs consecutive frames of each
    camera, with that camera's bounds, straight from the call's output"""
    import test_gpu_projection_domain as P
    torch, _ = _torch()
    params = (1000, 1.2, 8, fe.FAST_SCORE, 20)
    cams = []
    for W, H, seed in ((1280, 720, 41), (640, 480, 42)):
        base = textured_frame(W + 24, H + 24, seed=seed)
        cams.append(Frames(np.stack([np.ascontiguousarray(base[2 * i:2 * i + H, 3 * i:3 * i + W]) for i in range(3)])))
    ex = fe.ORBextractor(*params)
    try:
        out = multi(ex, cams)
        torch.cuda.synchronize()
    finally:
        ex.close()
    want = oracle(params, [f for c in cams for f in c.frames])
    same(out.host(), want, "frames")
    okps, odesc = [k for k, _ in want], [d for _, d in want]
    for c, cam in enumerate(cams):
        pairs = [(3 * c + 1, 3 * c), (3 * c + 2, 3 * c + 1)]
        for n in P.sbp_chain(out.kps, out.desc, out.cnt, out.cap, okps, odesc, pairs, cam.w, cam.h, cx=cam.w / 2, cy=cam.h / 2):
            assert n > 50, (cam.w, n)
