"""The CUDA extractor's orientation and steered BRIEF on the moment-designed frames of orient_domain_scenes.py: |m01| ==
|m10|, (0, 0), the half-disk bound, exact .5 ties of every sign and parity, angles where cosf / sinf would move a sample,
and keypoints 16-22 px from every edge at widths 0-3 mod 4 (samples outside the image, both patch-staging paths).

Every entry is compared with the oracle's default mode: angles as float32 bits, every other field and the descriptors
exactly.  Entries: ORBextractor on one frame and on a batch, orbfe_extract_batch_device in place (stride = width, and a
wider stride) and with ORBFE_INGEST_COPY=1; 1 and 8 levels.
"""
import numpy as np
import pytest

import oracle as O
import orb_slam_b200 as fe
import orient_domain_scenes as S

pytestmark = pytest.mark.gpu

NAMES = [s["name"] for s in S.scenes()]


def _scene(name):
    return next(s for s in S.scenes() if s["name"] == name)


def _oracle(img, nlevels):
    rc, k, d, _ = O.extract(O.make_params(S.nfeatures(nlevels), 1.2, nlevels, 1, S.FAST_TH), img)
    assert rc == 0
    return k, d


def _same(gk, gd, ok, od):
    assert len(gk) == len(ok), (len(gk), len(ok))
    for name in ("x", "y", "size", "response", "octave", "class_id"):
        assert np.array_equal(gk[name], ok[name]), name
    bad = np.flatnonzero(gk["angle"].view(np.uint32) != ok["angle"].view(np.uint32))
    assert len(bad) == 0, [(float(ok["x"][i]), float(ok["y"][i]), float(gk["angle"][i]), float(ok["angle"][i])) for i in bad[:5]]
    assert np.array_equal(gd, od)


def _extractor(nlevels):
    return fe.ORBextractor(S.nfeatures(nlevels), 1.2, nlevels, fe.FAST_SCORE, S.FAST_TH)


def _frames(name):
    """The scene and two mirrored copies (one geometry, so one batch)."""
    img = _scene(name)["img"]
    return np.stack([img, img[:, ::-1], img[::-1, :]])


@pytest.mark.parametrize("nlevels", [1, 8])
@pytest.mark.parametrize("name", NAMES)
def test_single_frame(gpu_required, name, nlevels):
    img = _scene(name)["img"]
    ex = _extractor(nlevels)
    try:
        gk, gd = ex(img)
    finally:
        ex.close()
    _same(gk, gd, *_oracle(img, nlevels))
    for x, y, _, _ in _scene(name)["kps"]:
        assert np.any((gk["octave"] == 0) & (gk["x"] == x) & (gk["y"] == y)), (x, y)


@pytest.mark.parametrize("nlevels", [1, 8])
@pytest.mark.parametrize("name", NAMES)
def test_batch(gpu_required, name, nlevels):
    frames = _frames(name)
    ex = _extractor(nlevels)
    try:
        kps, desc, cnt = ex.extract_batch(frames)
    finally:
        ex.close()
    for f in range(len(frames)):
        _same(kps[f, :cnt[f]], desc[f, :cnt[f]], *_oracle(frames[f], nlevels))


def _device_run(ex, frames, stride):
    """orbfe_extract_batch_device on frames laid out `stride` bytes per row (16-byte aligned rows and frames)."""
    import torch
    B, H, W = frames.shape
    host = np.full((B, H, stride), 0xA5, np.uint8)
    host[:, :, :W] = frames
    dev = torch.device("cuda", 0)
    buf = torch.from_numpy(host).to(dev)
    cap = int(ex.tables()[2].sum())
    d_kps = torch.zeros((B, cap, 28), dtype=torch.uint8, device=dev)
    d_desc = torch.zeros((B, cap, 32), dtype=torch.uint8, device=dev)
    d_cnt = torch.zeros((B,), dtype=torch.int32, device=dev)
    torch.cuda.synchronize()
    ex.extract_batch_device(buf.data_ptr(), W, H, stride, stride * H, B, d_kps.data_ptr(), d_desc.data_ptr(), d_cnt.data_ptr())
    ex.sync()
    k = d_kps.cpu().numpy().view(fe.KP_DTYPE).reshape(B, cap)
    d, c = d_desc.cpu().numpy(), d_cnt.cpu().numpy()
    return [(k[f, :c[f]], d[f, :c[f]]) for f in range(B)]


@pytest.mark.parametrize("nlevels", [1, 8])
@pytest.mark.parametrize("name", NAMES)
def test_device_ingest_paths(gpu_required, monkeypatch, name, nlevels):
    """In place with stride = width (where the width is a multiple of 16: level 0 is the caller's buffer and its pitch is
    the width), in place with a wider stride, and the copy path forced by ORBFE_INGEST_COPY=1."""
    frames = _frames(name)
    W = frames.shape[2]
    want = [_oracle(f, nlevels) for f in frames]
    strides = ([W] if W % 16 == 0 else []) + [(W + 15) // 16 * 16 + 64]
    ex = _extractor(nlevels)
    try:
        for stride in strides:
            for (gk, gd), (ok, od) in zip(_device_run(ex, frames, stride), want):
                _same(gk, gd, ok, od)
        monkeypatch.setenv("ORBFE_INGEST_COPY", "1")
        for (gk, gd), (ok, od) in zip(_device_run(ex, frames, strides[0]), want):
            _same(gk, gd, ok, od)
    finally:
        ex.close()
