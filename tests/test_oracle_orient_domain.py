"""The extractor's orientation and steered BRIEF at their float edges, on the CPU: the moment-designed frames of
orient_domain_scenes.py hold their facts, the numpy restatement equals the oracle (primitives and whole frames), every
named wrong variant changes the scenes that name it, and the reference's own ORBextractor gives the oracle's angles bit for
bit on every scene.
"""
import numpy as np
import pytest

import oracle as O
from oracle import ref as R
import orient_domain_scenes as S
from orb_slam_b200.synth import textured_frame

NAMES = [s["name"] for s in S.scenes()]


def _scene(name):
    return next(s for s in S.scenes() if s["name"] == name)


_RUNS = {}


def _run(name, nlevels=8, trig_mode=O.TRIG_RN):
    key = (name, nlevels, trig_mode)
    if key not in _RUNS:
        p = O.make_params(S.nfeatures(nlevels), 1.2, nlevels, 1, S.FAST_TH, trig_mode=trig_mode)
        rc, k, d, dump = O.extract(p, _scene(name)["img"], want_dump=True)
        assert rc == 0
        _RUNS[key] = (p, k, d, dump)
    return _RUNS[key]


def _designed(k, s):
    """Indices of the scene's designed keypoints in the oracle's output (each must be a level-0 keypoint)."""
    idx = []
    for x, y, _, _ in s["kps"]:
        hit = np.flatnonzero((k["octave"] == 0) & (k["x"] == x) & (k["y"] == y))
        assert len(hit) == 1, (s["name"], x, y)
        idx.append(int(hit[0]))
    return np.array(idx)


def _bits(a):
    return np.asarray(a, np.float32).view(np.uint32)


# ---------------------------------------------------------------------------------------------------------------------
# the restatement's primitives against the oracle's
# ---------------------------------------------------------------------------------------------------------------------
def test_fast_atan2_equals_the_oracle():
    """Random moments, both axes, |m01| == |m10| in every quadrant, +-1 around it, (0, 0) and the half-disk bound."""
    rng = np.random.default_rng(0)
    m = list(map(tuple, rng.integers(-700000, 700001, (3000, 2))))
    M = S.HALF_DISK_BOUND
    for k in (0, 1, 2, 777, 150000, M):
        for s1 in (1, -1):
            for s2 in (1, -1):
                m += [(s1 * k, s2 * k), (s1 * k, 0), (0, s2 * k), (s1 * (k + 1), s2 * k), (s1 * k, s2 * (k + 1)), (-1, M)]
    m = np.array(m)
    got = S.angle_of(m[:, 0], m[:, 1])
    want = np.array([O.fast_atan2(float(a), float(b)) for a, b in m], np.float32)
    assert np.array_equal(_bits(got), _bits(want))


@pytest.mark.parametrize("trig_mode,variant", [(O.TRIG_RN, None), (O.TRIG_LIBMF, "libmf")])
def test_brief_equals_the_oracle(trig_mode, variant):
    """The 512 rounded offsets and the descriptor against O.brief on a textured image, at random angles and at the
    designed keypoints' angles (ties and trig splits included)."""
    img = textured_frame(200, 160, seed=4)
    pad = O.reflect101_pad(img, S.E)
    rng = np.random.default_rng(1)
    ms = [(m01, m10) for s in S.scenes() for _, _, m01, m10 in s["kps"]]
    ang = np.concatenate([rng.uniform(0, 360, 200).astype(np.float32),
                          S.angle_of([m[0] for m in ms], [m[1] for m in ms])])
    xs, ys = rng.integers(20, 180, len(ang)), rng.integers(20, 140, len(ang))
    a, b = S.trig(ang, variant)
    rx, ry = S.offsets(a, b, variant)
    got = S.describe(pad, xs, ys, rx, ry)
    want = np.array([O.brief(pad, int(x), int(y), float(t), trig_mode) for x, y, t in zip(xs, ys, ang)])
    assert np.array_equal(got, want)


def test_fma32_is_one_rounding():
    """fma32 against exact rational arithmetic (round half to even), including x*y - fl(x*y)."""
    from fractions import Fraction
    rng = np.random.default_rng(2)
    x = rng.integers(-13, 13, 4000).astype(np.float32)
    y = rng.uniform(-1, 1, 4000).astype(np.float32)
    z = np.concatenate([rng.uniform(-20, 20, 2000).astype(np.float32), -(x[2000:] * y[2000:])])   # and the product's error
    got = S.fma32(x, y, z)
    for i in range(len(x)):
        exact = Fraction(float(x[i])) * Fraction(float(y[i])) + Fraction(float(z[i]))
        lo = np.float32(float(exact))
        cands = [np.nextafter(lo, np.float32(-np.inf)), lo, np.nextafter(lo, np.float32(np.inf))]
        errs = [abs(Fraction(float(c)) - exact) for c in cands]
        best = min(errs)
        ok = [c for c, e in zip(cands, errs) if e == best]
        if len(ok) > 1:
            ok = [c for c in ok if int(np.float32(c).view(np.uint32)) % 2 == 0]
        assert got[i] == ok[0], (x[i], y[i], z[i])


# ---------------------------------------------------------------------------------------------------------------------
# every scene holds its facts
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", NAMES)
def test_scene_holds_its_facts(name):
    """Designed moments on the oracle's level image, each designed keypoint in O.extract's output at level 0, and what
    each kind of scene is built for."""
    s = _scene(name)
    p, k, d, dump = _run(name)
    lev = dump["levels"][0]
    for x, y, m01, m10 in s["kps"]:
        assert O.ic_moments(lev, x, y) == (m01, m10), (name, x, y)
    idx = _designed(k, s)
    m = np.array([kp[2:] for kp in s["kps"]])
    ang = S.angle_of(m[:, 0], m[:, 1])
    assert np.array_equal(_bits(k["angle"][idx]), _bits(ang))
    a, b = S.trig(ang)
    if name == "zero_axes_diagonals":
        for want in [(0, 0), (0, 1), (1, 0), (0, -1), (-1, 0), (1, 1), (-1, -1), (1, -1), (-1, 1)]:
            assert want in [tuple(t) for t in m]
        assert np.sum(np.abs(m[:, 0]) == np.abs(m[:, 1])) >= 16
        assert np.sum(np.abs(np.abs(m[:, 0]) - np.abs(m[:, 1])) == 1) >= 6
        for pr in S.FMA_POLY_PAIRS:
            assert S.angle_of(*pr) != S.angle_of(*pr, variant="fma_poly")
    elif name == "saturated":
        M = S.HALF_DISK_BOUND
        assert [tuple(t) for t in m[:4]] == [(0, M), (M, 0), (0, -M), (-M, 0)]
        assert tuple(m[4]) == (-1, M) and np.float32(359.9998) < ang[4] < np.float32(360)
        diag = m[7:11]
        assert np.all(np.abs(diag[:, 0]) == np.abs(diag[:, 1])) and len({(np.sign(a_), np.sign(b_)) for a_, b_ in diag}) == 4
        assert sorted(abs(abs(int(a_)) - abs(int(b_))) for a_, b_ in m[11:15]) == [1, 1, 1, 1]
        assert tuple(m[15]) == (0, 0)
    elif name == "ties":
        got = S.ties(a, b)
        for cls, pairs in S.TIE_PAIRS.items():
            for pr in pairs:
                i = [tuple(t) for t in m].index(pr)
                assert got[i].get(cls, 0) >= 1, (cls, pr, got[i])
    elif name == "trig_split":
        al, bl = S.trig(ang, "libmf")
        rx, ry = S.offsets(a, b)
        lx, ly = S.offsets(al, bl)
        assert np.all(((rx != lx) | (ry != ly)).any(axis=1))
    elif name.startswith("border_"):
        W, H = s["W"], s["H"]
        n_out = S.outside_samples([kp[0] for kp in s["kps"]], [kp[1] for kp in s["kps"]], W, H, ang)
        near = np.array([min(x, y, W - 1 - x, H - 1 - y) for x, y, _, _ in s["kps"]])
        assert np.all(n_out[near <= 17] > 0) and np.all(n_out[near >= 18] == 0)
        assert set(near) == set(S.BORDER_D)
        xs = {x % 4 for x, y, _, _ in s["kps"] if min(x, W - 1 - x) in S.BORDER_D}
        assert xs == {0, 1, 2, 3}


# ---------------------------------------------------------------------------------------------------------------------
# the restatement equals the oracle, and every variant is caught
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", NAMES)
@pytest.mark.parametrize("nlevels,trig_mode,variant", [(8, O.TRIG_RN, None), (1, O.TRIG_RN, None), (8, O.TRIG_LIBMF, "libmf")])
def test_restatement_equals_extract(name, nlevels, trig_mode, variant):
    """Every keypoint of every level: angle (as bits) and descriptor of the restatement equal O.extract's."""
    p, k, d, dump = _run(name, nlevels, trig_mode)
    ang, desc = S.restate(p, dump, k, variant)
    assert np.array_equal(_bits(ang), _bits(k["angle"])) and np.array_equal(desc, d)


@pytest.mark.parametrize("name", NAMES)
def test_scene_names_the_variants_it_separates(name):
    """The variants that change a designed keypoint's angle or descriptor are exactly the ones the scene names."""
    s = _scene(name)
    p, k, d, dump = _run(name)
    idx = _designed(k, s)
    changed = []
    for v in S.VARIANTS:
        a2, d2 = S.restate(p, dump, k[idx], v)
        if not (np.array_equal(_bits(a2), _bits(k["angle"][idx])) and np.array_equal(d2, d[idx])):
            changed.append(v)
    assert tuple(changed) == s["variants"]


def test_every_variant_is_caught():
    assert {v for s in S.scenes() for v in s["variants"]} == set(S.VARIANTS)


# ---------------------------------------------------------------------------------------------------------------------
# the reference's own ORBextractor
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.skipif(not R.available(), reason="oracle/_ref is not built (the reference sources are absent)")
@pytest.mark.parametrize("name", NAMES)
def test_reference_angles_bit_for_bit(name):
    """src/ORBextractor.cc on the scenes: every keypoint and angle (as bits) equal to the oracle's with the literal
    nth_element retention.  Descriptors: the reference equals the oracle's TRIG_LIBMF mode on every scene (its translation
    unit calls cosf / sinf), and on the trig-split scene differs from the TRIG_RN mode the CUDA kernel implements."""
    img = _scene(name)["img"]
    rk, rd = R.extract(img, S.NF, 1.2, 8, 1, S.FAST_TH)
    desc = {}
    for tm in (O.TRIG_RN, O.TRIG_LIBMF):
        rc, k, d, _ = O.extract(O.make_params(S.NF, 1.2, 8, 1, S.FAST_TH, ties_mode=O.TIES_NTH_ELEMENT, trig_mode=tm), img)
        assert rc == 0 and len(k) == len(rk)
        for f in ("x", "y", "size", "response", "octave", "class_id"):
            assert np.array_equal(k[f], rk[f]), f
        assert np.array_equal(_bits(k["angle"]), _bits(rk["angle"]))
        desc[tm] = d
    assert np.array_equal(rd, desc[O.TRIG_LIBMF])
    assert np.array_equal(rd, desc[O.TRIG_RN]) == (name != "trig_split")
