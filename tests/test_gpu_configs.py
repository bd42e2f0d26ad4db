"""GPU parity at the BASELINE.json configurations that are not the bench line, plus full-size properties."""
import numpy as np
import pytest

import oracle as O
import orb_slam_b200 as fe
from orb_slam_b200 import matching as M, parallel as P
from orb_slam_b200.synth import textured_frame, shifted_frame, random_descriptors, noisy_copies

pytestmark = pytest.mark.gpu


def _same(gk, gd, ok, od):
    assert len(gk) == len(ok)
    for name in ("x", "y", "size", "response", "octave", "class_id"):
        assert np.array_equal(gk[name], ok[name]), name
    assert np.array_equal(gk["angle"].view(np.uint32), ok["angle"].view(np.uint32))
    assert np.array_equal(gd, od)


def test_config3_4k_12_levels(gpu_required):
    """configs[2]: 3840x2160, 4000 kp, 12 levels -- bit-exact against the oracle."""
    img = textured_frame(3840, 2160, seed=33)
    p = O.make_params(4000, 1.2, 12, 1, 20)
    rc, ok, od, _ = O.extract(p, img)
    assert rc == 0 and len(ok) == 4000
    ex = fe.ORBextractor(4000, 1.2, 12, fe.FAST_SCORE, 20)
    gk, gd = ex(img)
    _same(gk, gd, ok, od)
    ex.close()


def test_single_level_and_unsupported_geometry(gpu_required):
    img = textured_frame(640, 480, seed=4)
    p = O.make_params(300, 1.2, 1, 1, 20)
    rc, ok, od, _ = O.extract(p, img)
    assert rc == 0
    ex = fe.ORBextractor(300, 1.2, 1)
    gk, gd = ex(img)
    _same(gk, gd, ok, od)
    # degenerate geometry: oracle rc -2  <->  ORBFE_ERR_UNSUPPORTED, never a silent wrong answer
    tiny = np.zeros((40, 40), np.uint8)
    assert O.extract(O.make_params(300, 1.2, 1, 1, 20), tiny)[0] == -2
    with pytest.raises(fe.OrbfeError) as e:
        ex(tiny)
    assert e.value.code == fe.ORBFE_ERR_UNSUPPORTED
    ex.close()


@pytest.mark.parametrize("W,H,nf,nl", [(640, 480, 1000, 8), (1280, 720, 2000, 8), (641, 479, 500, 5)])
def test_harris_score_mode(gpu_required, W, H, nf, nl):
    """E6: scoreType == HARRIS_SCORE (ORBextractor.cc:616-620): retention ranks by the Harris response."""
    img = textured_frame(W, H, seed=W + 7)
    p = O.make_params(nf, 1.2, nl, 0, 20)
    rc, ok, od, _ = O.extract(p, img)
    assert rc == 0
    ex = fe.ORBextractor(nf, 1.2, nl, fe.HARRIS_SCORE, 20)
    gk, gd = ex(img)
    _same(gk, gd, ok, od)   # response compared bit-for-bit (float Harris value)
    assert len(gk) == nf and not np.array_equal(gk["response"], np.round(gk["response"]))
    ex.close()


def test_full_size_properties_1080p(gpu_required):
    """Size-independent properties at the bench geometry: determinism, batch == single, in-bounds, octave order."""
    f0 = textured_frame(1920, 1080, seed=9)
    f1 = shifted_frame(f0, 5, -3, seed=1)
    ex = fe.ORBextractor(2000, 1.2, 8)
    k0, d0 = ex(f0)
    k0b, d0b = ex(f0)
    assert np.array_equal(k0, k0b) and np.array_equal(d0, d0b)          # idempotent
    kps, desc, cnt = ex.extract_batch(np.stack([f0, f1, f0, f0]))
    assert list(cnt) == [2000, 2000, 2000, 2000]
    for i in (0, 2, 3):
        assert np.array_equal(kps[i], k0) and np.array_equal(desc[i], d0)  # slot independent
    assert np.all(np.diff(k0["octave"]) >= 0)
    s, _, q = ex.tables()
    for l in range(8):
        kl = k0[k0["octave"] == l]
        assert len(kl) == q[l]
        assert kl["x"].min() >= 16 * s[l] - 1e-3 and kl["x"].max() <= (ex.debug_level(0, l).shape[1] - 17) * s[l] + 1e-3
    # a 256-bit Hamming matrix is a metric: zero diagonal, symmetric, triangle inequality on a sample
    m = fe.ORBmatcher()
    D = m.hamming_dense(d0, d0).astype(np.int32)
    assert np.all(np.diag(D) == 0) and np.array_equal(D, D.T) and D.max() <= 256
    i, j, k = np.random.default_rng(0).integers(0, 2000, (3, 5000))
    assert np.all(D[i, k] <= D[i, j] + D[j, k])
    m.close()
    ex.close()


def test_config5_keyframe_db_sweep_sharded(gpu_required):
    """configs[4] primitive at reduced scale: 1 query set x keyframe DB, best/second per keyframe; sharding the
    DB rows over 1/2/4 'ranks' (shard_range) and concatenating gives the same answer as one sweep."""
    nq, nkf, per = 256, 40, 500
    q = random_descriptors(nq, 1)
    db = np.concatenate([noisy_copies(q[np.random.default_rng(g).integers(0, nq, per)], 0.12, 100 + g) for g in range(nkf)])
    m = fe.ORBmatcher()
    best, idx, second = m.knn2_groups(q, db, per)
    for g in (0, 17, 39):
        bd, bi, sd = O.knn2(q, db[g * per:(g + 1) * per])
        assert np.array_equal(best[g], bd) and np.array_equal(idx[g], bi) and np.array_equal(second[g], np.minimum(sd, 65535))
    for world in (2, 4):
        parts = []
        for r in range(world):
            lo, hi = P.shard_range(nkf, world, r)
            parts.append(m.knn2_groups(q, db[lo * per:hi * per], per))
        assert np.array_equal(np.concatenate([p[0] for p in parts]), best)
        assert np.array_equal(np.concatenate([p[1] for p in parts]), idx)
        assert np.array_equal(np.concatenate([p[2] for p in parts]), second)
    # loop-closure style score per keyframe: matches with best <= TH_LOW and best < 0.6 * second
    score = ((best <= 50) & (best < 0.6 * second)).sum(axis=1)
    assert score.max() > 0
    m.close()


def test_config4_cross_camera_initialization(gpu_required):
    """configs[3]: per-camera extraction, descriptor-block exchange (all-gather; world=1 here), then
    cross-camera SearchForInitialization against the oracle."""
    import torch
    import torch.distributed as dist
    Wc, Hc = 1280, 720
    cam0 = textured_frame(Wc, Hc, seed=71)
    cam1 = shifted_frame(cam0, 12, 4, seed=2)
    ex = fe.ORBextractor(2000, 1.2, 8)
    feats = [ex(c) for c in (cam0, cam1)]
    ex.close()
    blocks = []
    for k, d in feats:
        kp = np.zeros(2000, fe.KP_DTYPE); kp[:len(k)] = k
        dd = np.zeros((2000, 32), np.uint8); dd[:len(d)] = d
        blk = P.pack_block(torch, torch.from_numpy(kp.view(np.uint8).reshape(2000, 28)).cuda(), torch.from_numpy(dd).cuda(),
                           len(k), 2000, "cuda")
        blocks.append(P.allgather_blocks(torch, dist, blk)[0].cpu().numpy())
    (k0, d0), (k1, d1) = [P.unpack_block(b, fe.KP_DTYPE) for b in blocks]
    assert np.array_equal(k0, feats[0][0]) and np.array_equal(d1, feats[1][1])
    f0, f1 = M.FrameView(k0, d0, Wc, Hc), M.FrameView(k1, d1, Wc, Hc)
    o0, o1 = O.OracleFrame(k0, d0, Wc, Hc), O.OracleFrame(k1, d1, Wc, Hc)
    prev = np.stack([k0["x"], k0["y"]], axis=1).astype(np.float32)
    m = fe.ORBmatcher(0.9, True)
    n, m12, pv = M.search_for_initialization(m, f0, f1, prev, 100)
    n_o, m12_o, pv_o = O.search_for_initialization(o0, o1, prev, 100, nnratio=0.9, check_orientation=True)
    assert n == n_o and np.array_equal(m12, m12_o) and np.array_equal(pv, pv_o) and n > 50
    m.close()


@pytest.mark.parametrize("nf", [100, 60, 20])
def test_levels_with_an_empty_cell_grid(gpu_required, nf):
    """ORBextractor.cc:533-547: a level whose quota gives levelCols == 0 has empty cell vectors and yields no keypoints;
    the other levels run (the reference does not fail).  nfeatures=100 empties the last level, 60 the last four, 20 all."""
    img = textured_frame(640, 480, seed=3)
    p = O.make_params(nf, 1.2, 8, 1, 20)
    rc, ok, od, _ = O.extract(p, img)
    assert rc == 0
    ex = fe.ORBextractor(nf, 1.2, 8)
    gk, gd = ex(img)
    _same(gk, gd, ok, od)
    assert len(gk) == {100: 94, 60: 41, 20: 0}[nf]
    ex.close()
