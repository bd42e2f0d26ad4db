"""The candidate-set composition of extract_domain_scenes.py against oracle.extract, on the scenes the GPU domain tests use.

When every cell keeps every candidate, a level's keypoints are exactly the composition's set (the level images, the cell
windows with the reference's -3/+6 margins, cv::FAST + NMS per window, the <= 3 -> threshold-7 fallback).  This checks that
premise, and what each scene is built to show, against the oracle alone, so the GPU tests can rely on both.
"""
import numpy as np
import pytest

import oracle as O
import extract_domain_scenes as S

THRESHOLDS = [0, 1, 2, 6, 7, 8, 19, 21, 64, 127, 128, 200, 253, 254]


def _all_kept(p, img, W, H):
    rc, ok, _, dump = O.extract(p, img, want_dump=True)
    assert rc == 0
    per_level = []
    for l in range(p.nlevels):
        xyr, counts = S.level_candidates(p, dump, W, H, l)
        assert dump["n_level_kp"][l] == len(xyr), "level %d: retention cut candidates, the scene is too dense" % l
        assert np.array_equal(S.octave_triples(ok, l), S.to_output(p, l, xyr)), "level %d" % l
        per_level.append((xyr, counts))
    return ok, dump, per_level


SCENES = [("seam", g) for g in S.SEAM_GEOMETRIES] + [("count", th) for th in THRESHOLDS] + [("two_tone", th) for th in THRESHOLDS]


@pytest.mark.parametrize("kind,arg", SCENES, ids=["%s-%s" % (k, "x".join(map(str, a)) if isinstance(a, tuple) else a) for k, a in SCENES])
def test_composition_is_the_oracles_keypoint_set(kind, arg):
    if kind == "seam":
        W, H, nl = arg
        img, pairs = S.seam_scene(W, H, nl)
        p = O.make_params(S.SEAM_NF, 1.2, nl, 1, S.SEAM_TH)
        ok, dump, levels = _all_kept(p, img, W, H)
        keep, kinds = S.seam_expected(W, H, nl, pairs)
        assert min(kinds.values()) > 0, kinds
        got = {(int(x), int(y)) for x, y in zip(levels[0][0][:, 0], levels[0][0][:, 1])}
        assert got == keep
        return
    th = arg
    W, H = 320, 240
    if kind == "count":
        img, expect = S.count_scene(th, W, H)
        p = O.make_params(S.COUNT_NF, 1.2, S.COUNT_NL, 1, th)
        ok, dump, levels = _all_kept(p, img, W, H)
        xyr, counts = levels[0]
        assert counts[S.COUNT_CELL_A] == 3 and counts[S.COUNT_CELL_B] == 4
        assert dump["fallback"] == sum(1 for n in counts.values() if n <= 3) > 0
        g = O.cell_grid(p, 0, W, H, W, H)[1]
        cells = [((y - S.E) // g.cell_h, (x - S.E) // g.cell_w) for x, y, _ in xyr]
        for cell, n in expect.items():
            assert cells.count(cell) == n, (cell, n)
        assert len(xyr) == sum(expect.values())
    else:
        p = O.make_params(S.COUNT_NF, 1.2, S.COUNT_NL, 1, th)
        at_th = _all_kept(p, S.two_tone(th, th, W, H), W, H)
        # contrast th: not one corner at fastTh, every cell falls back; the threshold-7 pass finds the corners iff th > 7
        assert all(n == 0 for n in at_th[2][0][1].values())
        assert at_th[1]["fallback"] == len(at_th[2][0][1])
        assert (len(at_th[0]) > 0) == (th > 7)
        # contrast th + 1: corners at fastTh, except at th = 0 where their score is 0 and cv::FAST's strict NMS drops them
        above = _all_kept(p, S.two_tone(th, th + 1, W, H), W, H)
        assert (len(above[0]) > 0) == (th > 0)
