"""The CUDA extractor over its whole accepted domain, bit-exact against the oracle.

Every FAST threshold class (0 .. 254) on content whose ring differences sit exactly on the threshold; every candidate of a
level kept, with corners placed across every cell seam, FAST-tile seam and the detect border; the level-select kernel past
48 KB of shared memory and at the plan's refusal boundary; 16 and 32 levels, scale factors 1.01 .. 3.0; and every way a
frame is ingested by orbfe_extract_batch_device (in place, pitched, the 2-D copy path), with one handle switching between
them and the host entry.

Bar (as test_gpu_extract.py): x, y, size, response, octave, class_id equal; angle equal as float32 bits; descriptors equal.
"""
import numpy as np
import pytest

import oracle as O
import orb_slam_b200 as fe
import extract_domain_scenes as S
from orb_slam_b200.synth import textured_frame

pytestmark = pytest.mark.gpu

THRESHOLDS = [0, 1, 2, 6, 7, 8, 19, 21, 64, 127, 128, 200, 253, 254]


def _same(gk, gd, ok, od):
    assert len(gk) == len(ok), (len(gk), len(ok))
    for name in ("x", "y", "size", "response", "octave", "class_id"):
        assert np.array_equal(gk[name], ok[name]), name
    assert np.array_equal(gk["angle"].view(np.uint32), ok["angle"].view(np.uint32))
    assert np.array_equal(gd, od)


def _compare(img, nfeatures, nlevels, fast_th=20, sf=1.2, score=fe.FAST_SCORE):
    """Extract on the GPU and with the oracle; assert the bar.  Returns (gpu keypoints, params, oracle dump)."""
    p = O.make_params(nfeatures, sf, nlevels, score, fast_th)
    rc, ok, od, dump = O.extract(p, img, want_dump=True)
    assert rc == 0
    ex = fe.ORBextractor(nfeatures, sf, nlevels, score, fast_th)
    try:
        gk, gd = ex(img)
    finally:
        ex.close()
    _same(gk, gd, ok, od)
    return gk, p, dump


def _assert_all_kept(gk, p, dump, W, H):
    """Every level's keypoints are the complete FAST+NMS candidate set of the composition (nothing cut by retention)."""
    out = []
    for l in range(p.nlevels):
        xyr, counts = S.level_candidates(p, dump, W, H, l)
        assert dump["n_level_kp"][l] == len(xyr), "level %d: retention cut candidates" % l
        assert np.array_equal(S.octave_triples(gk, l), S.to_output(p, l, xyr)), "level %d" % l
        out.append((xyr, counts))
    return out


def _noise(W, H, seed):
    return np.random.default_rng(seed).integers(0, 256, (H, W), dtype=np.uint8)


# ---------------------------------------------------------------------------------------------------------------------
# 1. threshold domain
# ---------------------------------------------------------------------------------------------------------------------
def _threshold_cases(th, score):
    W, H = 320, 240
    for name, img in S.threshold_scenes(th).items():
        sparse = name in ("count", "two_tone_th", "two_tone_th1")
        nf, nl = (S.COUNT_NF, S.COUNT_NL) if sparse else (800, 3)
        gk, p, dump = _compare(img, nf, nl, th, score=score)
        if score != fe.FAST_SCORE:
            continue
        if sparse:
            (xyr, counts), = _assert_all_kept(gk, p, dump, W, H)
            if name == "count":
                # one cell at exactly 3 candidates at fastTh (falls back to threshold 7), one at exactly 4 (does not)
                assert counts[S.COUNT_CELL_A] == 3 and counts[S.COUNT_CELL_B] == 4
                assert dump["fallback"] > 0
                g = O.cell_grid(p, 0, W, H, W, H)[1]
                cells = [(int(y - S.E) // g.cell_h, int(x - S.E) // g.cell_w) for x, y in zip(gk["x"], gk["y"])]
                for cell, n in S.count_scene(th)[1].items():
                    assert cells.count(cell) == n, (cell, n)
            elif name == "two_tone_th":
                # contrast == th: no corner at fastTh anywhere, every cell falls back
                assert all(n == 0 for n in counts.values()) and dump["fallback"] == len(counts)
                assert (len(gk) > 0) == (th > 7)
            else:
                assert (len(gk) > 0) == (th > 0)
        elif name == "arcs":
            assert sum(dump["n_level_kp"]) > 0


@pytest.mark.parametrize("th", THRESHOLDS)
def test_fast_threshold_domain(gpu_required, th):
    """Ring differences at exactly th and th + 1 (arcs of 8, 9 and 10 pixels), two-tone corners of contrast th (none at
    fastTh: every cell takes the <= 3 -> threshold-7 fallback) and th + 1, binary 0/255 noise, a textured frame, and a
    scene with one cell at exactly 3 and one at exactly 4 candidates at fastTh."""
    _threshold_cases(th, fe.FAST_SCORE)


@pytest.mark.parametrize("th", [0, 7, 8, 254])
def test_fast_threshold_domain_harris(gpu_required, th):
    """The same scenes with HARRIS_SCORE retention."""
    _threshold_cases(th, fe.HARRIS_SCORE)


# ---------------------------------------------------------------------------------------------------------------------
# 2. every corner kept, at the seams
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("W,H,nl", S.SEAM_GEOMETRIES)
def test_every_corner_kept_across_seams(gpu_required, W, H, nl):
    """Detect areas with Wd mod 120 in {0, 1, 2, 118, 119} and Hd mod 62 in {0, 1, 61} (partial last FAST tiles), single-
    pixel corners in adjacent pairs across every cell seam, FAST-tile seam and the 16-px border, and enough features that
    every candidate is kept: each level's keypoints are exactly the composition's candidate set, and at level 0 a pair
    inside a cell resolves by strict NMS while a pair across a cell seam keeps both."""
    img, pairs = S.seam_scene(W, H, nl)
    gk, p, dump = _compare(img, S.SEAM_NF, nl, S.SEAM_TH)
    _assert_all_kept(gk, p, dump, W, H)
    keep, kinds = S.seam_expected(W, H, nl, pairs)
    assert min(kinds.values()) > 0, kinds
    k0 = gk[gk["octave"] == 0]
    assert {(int(x), int(y)) for x, y in zip(k0["x"], k0["y"])} == keep


# ---------------------------------------------------------------------------------------------------------------------
# 3. size limits
# ---------------------------------------------------------------------------------------------------------------------
def _level_select_smem(nf, nl, W, H, harris, sf=1.2):
    """Dynamic shared memory of the level-select kernel for this plan: a level keeps at most quota + 2 * cells + 64 keys;
    FAST retention sorts 8-byte keys in the next power of two, HARRIS holds 13 bytes per key plus 16."""
    p = O.make_params(nf, sf, nl, 1, 20)
    m = 0
    for l in range(nl):
        w, h = O.level_size(p, l, W, H)
        g = O.cell_grid(p, l, W, H, w, h)[1]
        m = max(m, p.quota[l] + 2 * g.n_cells + 64)
    if harris:
        return 13 * m + 16
    n2 = 1
    while n2 < m:
        n2 <<= 1
    return 8 * n2


@pytest.mark.parametrize("W,H,nf,nl,score", [(1600, 1200, 7000, 1, fe.FAST_SCORE), (1280, 720, 15000, 2, fe.FAST_SCORE),
                                             (640, 480, 3000, 1, fe.HARRIS_SCORE), (1600, 1200, 5000, 1, fe.HARRIS_SCORE)])
def test_level_select_beyond_48k_shared_memory(gpu_required, W, H, nf, nl, score):
    assert _level_select_smem(nf, nl, W, H, score == fe.HARRIS_SCORE) > 48 * 1024
    gk, _, _ = _compare(_noise(W, H, nf), nf, nl, fast_th=10, score=score)
    assert len(gk) == nf


@pytest.mark.parametrize("score", [fe.FAST_SCORE, fe.HARRIS_SCORE])
def test_level_select_refusal_boundary(gpu_required, score):
    """The smallest nfeatures (one level, 1600x1200) whose level-select footprint exceeds 200 KB is refused with
    ORBFE_ERR_UNSUPPORTED; one fewer runs and matches the oracle.

    Known limit: the oracle (like the reference) runs the refused count; the library does not."""
    W, H = 1600, 1200
    harris = score == fe.HARRIS_SCORE
    nf = next(n for n in range(8000, 20000) if _level_select_smem(n, 1, W, H, harris) > 200 * 1024)
    img = _noise(W, H, 11)
    assert O.extract(O.make_params(nf, 1.2, 1, score, 10), img)[0] == 0
    ex = fe.ORBextractor(nf, 1.2, 1, score, 10)
    with pytest.raises(fe.OrbfeError) as e:
        ex(img)
    ex.close()
    assert e.value.code == fe.ORBFE_ERR_UNSUPPORTED and "level-select" in str(e.value)
    gk, _, _ = _compare(img, nf - 1, 1, fast_th=10, score=score)
    assert len(gk) == nf - 1


@pytest.mark.parametrize("W,H,nl,sf", [(640, 480, 16, 1.01), (640, 480, 16, 1.05), (640, 480, 32, 1.01), (640, 480, 32, 1.05),
                                        (640, 480, 3, 2.0), (1280, 960, 4, 2.0), (640, 480, 2, 3.0), (1280, 960, 3, 3.0)])
def test_level_counts_and_scale_factors(gpu_required, W, H, nl, sf):
    """Up to the 32-level maximum at small scale factors; scale factors 2.0 and 3.0 (the generic resize path)."""
    gk, _, dump = _compare(textured_frame(W, H, seed=21), 1000, nl, sf=sf)
    assert all(n > 0 for n in dump["n_level_kp"])


@pytest.mark.parametrize("nl,sf,oracle_rc", [(4, 2.0, 0), (3, 3.0, 0), (5, 2.0, -2), (4, 3.0, -2)])
def test_refused_level_geometries(gpu_required, nl, sf, oracle_rc):
    """640x480 pyramids whose last level the library refuses: ORBFE_ERR_UNSUPPORTED, never a result.

    Known limits: 4 levels at 2.0 and 3 levels at 3.0, which the oracle runs.  Their last level's cells (16x7, 13x6 px)
    are too small for the FAST tile, which counts candidates for at most 64 cells.  With 5 levels at 2.0 and 4 at 3.0 the
    oracle refuses too: the last level's cell grid does not tile its detect area."""
    img = textured_frame(640, 480, seed=21)
    assert O.extract(O.make_params(1000, sf, nl, 1, 20), img)[0] == oracle_rc
    ex = fe.ORBextractor(1000, sf, nl)
    with pytest.raises(fe.OrbfeError) as e:
        ex(img)
    ex.close()
    assert e.value.code == fe.ORBFE_ERR_UNSUPPORTED


# ---------------------------------------------------------------------------------------------------------------------
# 4. frame ingest and handle state
# ---------------------------------------------------------------------------------------------------------------------
def _layout(frames, off, stride, frame_stride, fill=0xA5):
    """Host bytes holding `frames` at byte offset `off`, rows `stride` apart, frames `frame_stride` apart; padding = fill."""
    B, H, W = frames.shape
    buf = np.full(off + B * frame_stride + 64, fill, np.uint8)
    for f in range(B):
        base = off + f * frame_stride
        buf[base:base + stride * H].reshape(H, stride)[:, :W] = frames[f]
    return buf


class _Dev:
    """Device buffers for orbfe_extract_batch_device (torch allocations, synchronised around every call: the library
    enqueues on its own non-blocking stream)."""

    def __init__(self, torch):
        self.torch = torch
        self.dev = torch.device("cuda", 0)

    def upload(self, host):
        return self.torch.from_numpy(host).to(self.dev)

    def run(self, ex, ptr, W, H, stride, frame_stride, B):
        t = self.torch
        cap = int(ex.tables()[2].sum())
        d_kps = t.zeros((B, cap, 28), dtype=t.uint8, device=self.dev)
        d_desc = t.zeros((B, cap, 32), dtype=t.uint8, device=self.dev)
        d_cnt = t.zeros((B,), dtype=t.int32, device=self.dev)
        t.cuda.synchronize()
        ex.extract_batch_device(ptr, W, H, stride, frame_stride, B, d_kps.data_ptr(), d_desc.data_ptr(), d_cnt.data_ptr())
        ex.sync()
        k = d_kps.cpu().numpy().view(fe.KP_DTYPE).reshape(B, cap)
        d, c = d_desc.cpu().numpy(), d_cnt.cpu().numpy()
        return [(k[f, :c[f]], d[f, :c[f]]) for f in range(B)]


def _oracle(frames, nf=1000, nl=8):
    out = []
    for img in frames:
        rc, ok, od, _ = O.extract(O.make_params(nf, 1.2, nl, 1, 20), img)
        assert rc == 0
        out.append((ok, od))
    return out


def _same_all(got, want):
    assert len(got) == len(want)
    for (gk, gd), (ok, od) in zip(got, want):
        _same(gk, gd, ok, od)


def test_ingest_paths_agree(gpu_required, monkeypatch):
    """The same frames through every ingest path of orbfe_extract_batch_device: in place (aligned, and pitched with
    stride = W + 64 and a frame stride past stride * H), the 2-D copy (base 1, 8 and 15 bytes off alignment; stride W + 1;
    a frame stride past stride * H) and ORBFE_INGEST_COPY=1.  All give the oracle's answer per frame."""
    import torch
    D = _Dev(torch)
    W, H, B = 640, 480, 3
    frames = np.stack([textured_frame(W, H, seed=60 + i) for i in range(B)])
    want = _oracle(frames)
    ex = fe.ORBextractor(1000, 1.2, 8)
    pitch = (W + 64 + 15) // 16 * 16
    layouts = [(0, W, W * H), (0, pitch, pitch * H + 4096),                          # in place
               (1, W, W * H), (8, W, W * H), (15, W, W * H), (0, W + 1, (W + 1) * H),  # 2-D copy
               (8, W + 1, (W + 1) * H + 3)]                                            # 2-D copy, frame by frame
    for off, stride, fs in layouts:
        buf = D.upload(_layout(frames, off, stride, fs))
        _same_all(D.run(ex, buf.data_ptr() + off, W, H, stride, fs, B), want)
    monkeypatch.setenv("ORBFE_INGEST_COPY", "1")
    buf = D.upload(_layout(frames, 0, W, W * H))
    _same_all(D.run(ex, buf.data_ptr(), W, H, W, W * H, B), want)
    ex.close()


def test_one_handle_across_ingest_paths_and_plans(gpu_required):
    """One handle: device in place (buffer A) -> device copy -> host extract_batch -> device in place on buffer B with
    another pitch -> device in place on A again -> a geometry change (plan rebuild) -> a batch larger than the first plan's.
    Buffer A is overwritten with other frames (and stays allocated) after its first use, so a level 0 left pointing at A
    gives wrong keypoints instead of reading freed memory."""
    import torch
    D = _Dev(torch)
    W, H, B = 640, 480, 2
    fr = {k: np.stack([textured_frame(W, H, seed=100 + 10 * k + i) for i in range(B)]) for k in range(5)}
    ex = fe.ORBextractor(1000, 1.2, 8)
    A = D.upload(_layout(fr[0], 0, W, W * H))
    _same_all(D.run(ex, A.data_ptr(), W, H, W, W * H, B), _oracle(fr[0]))
    A.copy_(D.upload(_layout(fr[4], 0, W, W * H)))
    C = D.upload(_layout(fr[1], 8, W, W * H))
    _same_all(D.run(ex, C.data_ptr() + 8, W, H, W, W * H, B), _oracle(fr[1]))
    kps, desc, cnt = ex.extract_batch(fr[2])
    _same_all([(kps[f, :cnt[f]], desc[f, :cnt[f]]) for f in range(B)], _oracle(fr[2]))
    pitch = W + 128
    Bb = D.upload(_layout(fr[3], 0, pitch, pitch * H))
    _same_all(D.run(ex, Bb.data_ptr(), W, H, pitch, pitch * H, B), _oracle(fr[3]))
    _same_all(D.run(ex, A.data_ptr(), W, H, W, W * H, B), _oracle(fr[4]))
    # geometry change: the plan is rebuilt
    W2, H2 = 752, 480
    g = np.stack([textured_frame(W2, H2, seed=150 + i) for i in range(B)])
    G = D.upload(_layout(g, 0, W2, W2 * H2))
    A.fill_(0)
    _same_all(D.run(ex, G.data_ptr(), W2, H2, W2, W2 * H2, B), _oracle(g))
    # a batch larger than the plan's: rebuilt again; then the copy path on the new plan
    B2 = 5
    g2 = np.stack([textured_frame(W2, H2, seed=160 + i) for i in range(B2)])
    G.fill_(0)
    G2 = D.upload(_layout(g2, 0, W2, W2 * H2))
    want2 = _oracle(g2)
    _same_all(D.run(ex, G2.data_ptr(), W2, H2, W2, W2 * H2, B2), want2)
    G3 = D.upload(_layout(g2, 1, W2 + 1, (W2 + 1) * H2))
    _same_all(D.run(ex, G3.data_ptr() + 1, W2, H2, W2 + 1, (W2 + 1) * H2, B2), want2)
    ex.close()


def mixed_frames(W=640, H=480, B=64):
    """B frames of mixed content: flat, binary 0/255 noise, two-tone single-pixel corners, textured, and frame 17 all zero"""
    frames = []
    for i in range(B):
        kind = i % 4
        if kind == 0:
            frames.append(np.full((H, W), (37 * i) % 256, np.uint8))
        elif kind == 1:   # binary 0/255 noise, dense and sparse
            density = 0.5 if i % 8 == 1 else 0.02
            frames.append(((np.random.default_rng(i).random((H, W)) < density) * 255).astype(np.uint8))
        elif kind == 2:
            frames.append(S.two_tone(20, 21 + i, W, H))
        else:
            frames.append(textured_frame(W, H, seed=200 + i))
    frames[17] = np.zeros((H, W), np.uint8)
    return np.stack(frames)


def test_mixed_content_batch_of_64(gpu_required):
    """One call over 64 frames of mixed content at 640x480: flat, binary 0/255 noise, two-tone single-pixel corners,
    textured, and one frame all zero; per frame equal to the oracle."""
    import torch
    D = _Dev(torch)
    W, H, B = 640, 480, 64
    frames = mixed_frames(W, H, B)
    want = _oracle(frames)
    assert sum(len(k) == 0 for k, _ in want) >= 16 and sum(len(k) == 1000 for k, _ in want) >= 16
    ex = fe.ORBextractor(1000, 1.2, 8)
    buf = D.upload(_layout(frames, 0, W, W * H))
    _same_all(D.run(ex, buf.data_ptr(), W, H, W, W * H, B), want)
    ex.close()
