"""GPU parity: liborbfe.so (through the C-ABI) against the CPU oracle on the same seeded inputs.

Bar: pixel coordinates, octave and 32-byte descriptors bit-exact; IC_Angle equal as float32 bits.
"""
import numpy as np
import pytest

import oracle as O
import orb_slam_b200 as fe
from orb_slam_b200.synth import textured_frame

pytestmark = pytest.mark.gpu


def _compare(img, nfeatures, nlevels, fast_th=20, sf=1.2, check_levels=True):
    H, W = img.shape
    p = O.make_params(nfeatures, sf, nlevels, 1, fast_th)
    rc, ok, od, dump = O.extract(p, img, want_dump=True)
    assert rc == 0
    ex = fe.ORBextractor(nfeatures, sf, nlevels, fe.FAST_SCORE, fast_th)
    gk, gd = ex(img)
    if check_levels:
        for l in range(nlevels):
            lev = dump["levels"][l][O.EDGE:-O.EDGE, O.EDGE:-O.EDGE]
            assert np.array_equal(ex.debug_level(0, l, False), lev), "pyramid level %d differs" % l
            if dump["n_level_kp"][l] > 0:
                blr = dump["blurred"][l][O.EDGE:-O.EDGE, O.EDGE:-O.EDGE]
                assert np.array_equal(ex.debug_level(0, l, True), blr), "blurred level %d differs" % l
    assert len(gk) == len(ok), (len(gk), len(ok))
    # canonical order is defined (level, cell row-major, raster): compare element-wise
    for name in ("x", "y", "size", "response", "octave", "class_id"):
        assert np.array_equal(gk[name], ok[name]), name
    assert np.array_equal(gk["angle"].view(np.uint32), ok["angle"].view(np.uint32))
    assert np.array_equal(gd, od)
    ex.close()
    return len(gk)


def test_config1_640x480(gpu_required):
    n = _compare(textured_frame(640, 480, seed=1), 1000, 8)
    assert n == 1000


def test_1080p_2000(gpu_required):
    n = _compare(textured_frame(1920, 1080, seed=2), 2000, 8)
    assert n == 2000


@pytest.mark.parametrize("W,H,nf,nl,th", [(752, 480, 1000, 8, 20), (641, 479, 500, 5, 20), (1280, 720, 2000, 8, 20),
                                            (640, 480, 1000, 8, 7), (640, 480, 1000, 8, 5), (333, 257, 300, 4, 20),
                                            (640, 480, 2000, 8, 20), (752, 480, 4000, 8, 20)])
def test_geometries(gpu_required, W, H, nf, nl, th):
    _compare(textured_frame(W, H, seed=W + H), nf, nl, fast_th=th)


def test_other_scale_factors(gpu_required):
    """scale factors on both sides of the resize kernel's fast-path limit (4/3)"""
    _compare(textured_frame(640, 480, seed=12), 800, 5, sf=1.1)
    _compare(textured_frame(640, 480, seed=13), 600, 4, sf=1.5)
    _compare(textured_frame(800, 600, seed=14), 500, 3, sf=1.7)


def test_flat_and_noise(gpu_required):
    flat = np.full((480, 640), 77, np.uint8)
    assert _compare(flat, 1000, 8) == 0
    rng = np.random.default_rng(5)
    noise = rng.integers(0, 256, (480, 640), dtype=np.uint8)
    _compare(noise, 1000, 8)
    grad = (np.add.outer(np.arange(480), np.arange(640)) % 256).astype(np.uint8)
    _compare(grad, 1000, 8)
    chk = (((np.arange(480)[:, None] // 8) + (np.arange(640)[None, :] // 8)) % 2 * 200 + 20).astype(np.uint8)
    _compare(chk, 1000, 8)


def test_batch_matches_single(gpu_required):
    frames = np.stack([textured_frame(640, 480, seed=10 + i) for i in range(5)])
    ex = fe.ORBextractor(1000, 1.2, 8)
    kps, desc, counts = ex.extract_batch(frames)
    for i in range(5):
        k1, d1 = ex(frames[i])
        assert counts[i] == len(k1)
        assert np.array_equal(kps[i, :counts[i]], k1)
        assert np.array_equal(desc[i, :counts[i]], d1)
    ex.close()


def test_strided_input_and_empty(gpu_required):
    big = textured_frame(800, 600, seed=3)
    view = big[50:530, 100:740]  # 640x480 view with stride 800
    ex = fe.ORBextractor(1000, 1.2, 8)
    k1, d1 = ex(view)
    k2, d2 = ex(np.ascontiguousarray(view))
    assert np.array_equal(k1, k2) and np.array_equal(d1, d2)
    k0, d0 = ex(np.zeros((0, 0), np.uint8))
    assert len(k0) == 0 and d0.shape == (0, 32)
    ex.close()


@pytest.mark.parametrize("env", [{}, {"ORBFE_PDL": "0"}])
def test_alternate_kernel_paths(gpu_required, env, monkeypatch):
    """The kernels launched with and without programmatic dependent launch (ORBFE_PDL=0) produce the same bits as the
    oracle, on a second odd geometry with fewer levels and a FAST threshold between 7 and 20."""
    for k, v in env.items():
        monkeypatch.setenv(k, v)
    _compare(textured_frame(752, 480, seed=3), 1000, 8)
    _compare(textured_frame(641, 479, seed=6), 700, 6, fast_th=12)


def test_phased_batch_mode_matches_chunked(gpu_required):
    """orbfe_extractor_set_batch_mode: the two schedules of a batch give identical results."""
    frames = np.stack([textured_frame(640, 480, seed=40 + i) for i in range(12)])
    ex = fe.ORBextractor(800, 1.2, 8)
    k0, d0, c0 = ex.extract_batch(frames)
    ex.set_batch_mode(1)
    k1, d1, c1 = ex.extract_batch(frames)
    assert np.array_equal(c0, c1) and c0.min() > 300
    for f in range(len(frames)):
        assert np.array_equal(k0[f, :c0[f]], k1[f, :c1[f]]) and np.array_equal(d0[f, :c0[f]], d1[f, :c1[f]])
    with pytest.raises(fe.OrbfeError):
        ex.set_batch_mode(7)
    ex.close()


def test_random_geometries_and_extreme_contrast(gpu_required):
    """A seeded sweep over image sizes / feature counts / level counts / thresholds, on content that reaches both ends of the u8
    range (binary 0/255 noise, saturated blobs on texture): the FAST arc network runs part of its min/max on the FMA pipe as
    fp16-subnormal arithmetic, which must be exact for every value 0..255 and every difference of two of them."""
    rng = np.random.default_rng(2024)
    for it in range(10):
        W = int(rng.integers(200, 1100))
        H = int(rng.integers(160, 800))
        nl = int(rng.integers(2, 9))
        nf = int(rng.integers(150, 2500))
        th = int(rng.choice([5, 7, 12, 20, 35]))
        kind = it % 3
        if kind == 0:
            img = textured_frame(W, H, seed=900 + it)
            for _ in range(6):   # saturated and black blobs
                x0, y0 = int(rng.integers(0, W - 40)), int(rng.integers(0, H - 40))
                img[y0:y0 + int(rng.integers(5, 40)), x0:x0 + int(rng.integers(5, 40))] = int(rng.choice([0, 255]))
        elif kind == 1:
            img = (rng.integers(0, 2, (H, W), dtype=np.uint8) * 255).astype(np.uint8)   # binary noise: every ring value is 0 or 255
        else:
            img = rng.integers(0, 256, (H, W), dtype=np.uint8)
            img[::7, ::5] = 255
            img[3::11, 2::9] = 0
        img = np.ascontiguousarray(img)
        rc = O.extract(O.make_params(nf, 1.2, nl, 1, th), img)[0]
        if rc == -2:
            # a cell grid the reference itself cannot run ((cols-1)*cellW reaches past the image: cv::Mat::colRange throws,
            # ORBextractor.cc:599): the oracle and the library both refuse it
            ex = fe.ORBextractor(nf, 1.2, nl, fe.FAST_SCORE, th)
            with pytest.raises(fe.OrbfeError):
                ex(img)
            ex.close()
            continue
        _compare(img, nf, nl, fast_th=th, check_levels=False)
