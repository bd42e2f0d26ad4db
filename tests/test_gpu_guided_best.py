"""orbfe_guided_best (the best-candidate search of Fuse and SearchBySim3) on the fused kernel, index for index against the
oracle's plain loop: ties for the minimum (the first candidate in GetFeaturesInArea order wins), the distance threshold,
empty windows / frames / query sets, the octave filters, windows on grid-cell seams and image edges, and calls with more
queries than one launch holds (run in consecutive launches), also with the candidates in the global scratch.  The same
query chunking for orbfe_guided_search without the rotation histogram, and the histogram's refusal at that size.  The CPU
part: bad arguments are rejected before the matcher handle is used, each with a message."""
import ctypes as C

import numpy as np
import pytest

import oracle as O
import orb_slam_b200 as fe
from orb_slam_b200 import matching as M
from orb_slam_b200.synth import noisy_copies, random_descriptors

W, H = 640, 480          # cells of 10 x 10 px
LIMIT = 24826            # queries one launch holds in a 2000-feature frame (sbp_smem_fixed_bytes + 16 KB <= 220 KB)


def _kps(x, y, octave, angle=0.0):
    k = np.zeros(len(x), fe.KP_DTYPE)
    k["x"], k["y"], k["octave"], k["angle"] = x, y, octave, angle
    k["size"], k["response"], k["class_id"] = 31.0, 1.0, -1
    return k


def _views(k, d, nlevels=8):
    return M.FrameView(k, d, W, H, nlevels=nlevels), O.OracleFrame(k, d, W, H, nlevels=nlevels)


def _flip(d, nbits, rng):
    """d with `nbits` distinct bits flipped: at Hamming distance nbits."""
    bits = np.unpackbits(d.copy())
    idx = rng.choice(256, nbits, replace=False)
    bits[idx] ^= 1
    return np.packbits(bits)


def _same(m, v, o, qu, qv, qr, lo, hi, qd, th):
    got = M.guided_best(m, v, qu, qv, qr, lo, hi, qd, th)
    want = O.guided_best(o, qu, qv, qr, lo, hi, qd, th)
    assert np.array_equal(got, want), np.flatnonzero(got != want)[:10]
    return got


def _random_scene(n, nq, seed, r=(2.0, 30.0), octaves=8):
    """A frame of n features and nq queries near its features, with noisy copies of their descriptors."""
    rng = np.random.default_rng(seed)
    k = _kps(rng.uniform(0, W - 1, n), rng.uniform(0, H - 1, n), rng.integers(0, octaves, n), rng.uniform(0, 360, n))
    d = random_descriptors(n, seed + 1)
    src = rng.integers(0, max(n, 1), nq)
    qu = (k["x"][src] + rng.normal(0, 2, nq)).astype(np.float32) if n else rng.uniform(0, W, nq).astype(np.float32)
    qv = (k["y"][src] + rng.normal(0, 2, nq)).astype(np.float32) if n else rng.uniform(0, H, nq).astype(np.float32)
    qr = rng.uniform(*r, nq).astype(np.float32)
    lv = rng.integers(0, octaves, nq).astype(np.int32)
    qd = noisy_copies(d[src], 0.12, seed + 2) if n else random_descriptors(nq, seed + 2)
    return k, d, qu, qv, qr, (lv - 1).astype(np.int32), lv, qd


# ---- CPU: argument checks ----

def test_guided_best_rejects_bad_arguments_before_the_handle():
    """Every rejection is ORBFE_ERR_ARG with orbfe_last_error naming orbfe_guided_best, and happens before the handle (a
    zeroed host buffer here, never a real matcher) is used."""
    L = M._bind()
    buf = C.create_string_buffer(256)
    h = C.c_void_p(C.addressof(buf))
    bufs = [C.create_string_buffer(64) for _ in range(9)]
    p = [C.c_void_p(C.addressof(b)) for b in bufs]
    qu, qv, qr, lo, hi, qd, out, keys, desc = p

    def view(n=4, keys_un=keys, d=desc):
        v = M._FrameViewC()
        v.n, v.keys_un, v.desc = n, keys_un, d
        v.min_x, v.min_y, v.max_x, v.max_y, v.grid_inv_w, v.grid_inv_h = 0.0, 0.0, float(W), float(H), 0.1, 0.1
        v.nlevels, v.scale_factors = 1, None
        return v

    def call(m=h, f="view", nq=3, q=None, best=out):
        f = view() if f == "view" else f
        q = [qu, qv, qr, lo, hi, qd] if q is None else q
        return L.orbfe_guided_best(m, None if f is None else C.byref(f), nq, *q, 50, best)

    def other_error():   # a rejection by another entry, so that each check below sees its own message
        assert L.orbfe_guided_search(None, None, 0, None, None, None, None, None, None, None, 0, 0.8, 50, 0, None, None) == fe.ORBFE_ERR_ARG
        assert fe.lib().orbfe_last_error().startswith(b"orbfe_guided_search")

    cases = [dict(m=None), dict(f=None), dict(nq=-1), dict(best=None), dict(f=view(n=-1)), dict(f=view(keys_un=None)),
             dict(f=view(d=None))]
    for k in range(6):
        q = [qu, qv, qr, lo, hi, qd]
        q[k] = None
        cases.append(dict(q=q))
    for kw in cases:
        other_error()
        assert call(**kw) == fe.ORBFE_ERR_ARG, kw
        assert fe.lib().orbfe_last_error().startswith(b"orbfe_guided_best"), kw
    # accepted without reading a pointer: no queries and no features never reach the device
    assert call(f=view(n=0, keys_un=None, d=None), nq=0, q=[None] * 6) == fe.ORBFE_OK


# ---- GPU: against the oracle ----

@pytest.mark.gpu
def test_ties_go_to_the_first_candidate_in_enumeration_order(gpu_required):
    """Candidates at equal distance in one window: the first in GetFeaturesInArea order (cell column, then row, then index)
    wins, which here is never the lowest feature index."""
    rng = np.random.default_rng(1)
    base = random_descriptors(1, 5)[0]
    # 10-px cells: feature 0 is in cell column 13, features 1 and 2 share cell (11, 10); all three at distance 6
    x = np.array([125.0, 114.6, 113.0, 300.0], np.float32)
    y = np.array([100.0, 101.0, 99.0, 300.0], np.float32)
    k = _kps(x, y, 0)
    d = np.stack([_flip(base, 6, rng), _flip(base, 6, rng), _flip(base, 6, rng), base])
    v, o = _views(k, d)
    m = fe.ORBmatcher(0.8, False)
    one = lambda a, t: np.array([a], t)
    got = _same(m, v, o, one(120.0, np.float32), one(100.0, np.float32), one(10.0, np.float32), one(-1, np.int32), one(-1, np.int32),
                base[None], 50)
    assert got[0] == 1     # column 11 before column 13, and inside cell (11, 10) the lower index
    # many ties: descriptors drawn from four patterns, so most windows hold several candidates at the minimum
    k, d, qu, qv, qr, lo, hi, qd = _random_scene(2000, 3000, seed=2, r=(5.0, 40.0))
    pats = random_descriptors(4, 9)
    d = pats[np.random.default_rng(3).integers(0, 4, 2000)]
    qd = pats[np.random.default_rng(4).integers(0, 4, 3000)]
    v, o = _views(k, d)
    got = _same(m, v, o, qu, qv, qr, np.full(3000, -1, np.int32), np.full(3000, -1, np.int32), qd, 50)
    assert (got >= 0).sum() > 2500
    m.close()


@pytest.mark.gpu
def test_threshold_is_inclusive(gpu_required):
    """best == th_dist is kept, th_dist one lower drops it."""
    rng = np.random.default_rng(6)
    base = random_descriptors(1, 7)[0]
    for dist in (0, 1, 37, 50, 100, 256):
        d = np.stack([_flip(base, dist, rng), _flip(base, min(dist + 3, 256), rng)])
        k = _kps(np.array([200.0, 203.0], np.float32), np.array([200.0, 198.0], np.float32), 0)
        v, o = _views(k, d)
        m = fe.ORBmatcher(0.8, False)
        q = lambda a, t: np.array([a], t)
        args = (q(201.0, np.float32), q(200.0, np.float32), q(8.0, np.float32), q(-1, np.int32), q(-1, np.int32), base[None])
        assert _same(m, v, o, *args, dist)[0] == 0
        if dist > 0:
            assert _same(m, v, o, *args, dist - 1)[0] == -1
        m.close()


@pytest.mark.gpu
def test_empty_windows_frames_and_query_sets(gpu_required):
    """Windows off the image or over no feature give -1; an empty frame gives -1 everywhere; no queries is a no-op."""
    m = fe.ORBmatcher(0.8, False)
    k, d, qu, qv, qr, lo, hi, qd = _random_scene(500, 400, seed=8)
    qu[:100] += np.float32(2000.0)           # right of the image
    qv[100:200] -= np.float32(2000.0)        # above it
    qr[200:300] = np.float32(0.01)           # tiny windows, mostly empty
    v, o = _views(k, d)
    got = _same(m, v, o, qu, qv, qr, lo, hi, qd, 100)
    assert (got[:200] == -1).all() and (got[300:] >= 0).any()
    v0, o0 = _views(k[:0], d[:0])
    assert (_same(m, v0, o0, qu, qv, qr, lo, hi, qd, 100) == -1).all()
    e = np.zeros(0, np.float32)
    ei = np.zeros(0, np.int32)
    assert len(_same(m, v, o, e, e, e, ei, ei, qd[:0], 100)) == 0
    m.close()


@pytest.mark.gpu
def test_octave_filters(gpu_required):
    """(-1, -1) = every octave, (lv - 1, lv) with lv = 0 = octave 0 only, (lv, lv) = one level, and a one-level frame."""
    m = fe.ORBmatcher(0.8, False)
    k, d, qu, qv, qr, lo, hi, qd = _random_scene(2000, 2000, seed=12, r=(10.0, 40.0))
    v, o = _views(k, d)
    n = len(qu)
    for lo_, hi_ in ((np.full(n, -1), np.full(n, -1)), (np.full(n, -1), np.zeros(n)), (hi, hi), (lo, hi)):
        got = _same(m, v, o, qu, qv, qr, np.asarray(lo_, np.int32), np.asarray(hi_, np.int32), qd, 80)
        assert (got >= 0).sum() > 100
    k1 = k.copy()
    k1["octave"] = 0
    v1, o1 = _views(k1, d, nlevels=1)
    _same(m, v1, o1, qu, qv, qr, np.full(n, -1, np.int32), np.zeros(n, np.int32), qd, 80)
    m.close()


@pytest.mark.gpu
def test_windows_on_cell_seams_and_image_edges(gpu_required):
    """Features and window centres on cell boundaries (multiples of 5 px: seams and cell centres), radii that end exactly
    on a seam, and windows that reach past every image edge."""
    rng = np.random.default_rng(13)
    n = 1500
    x = (rng.integers(0, W // 5, n) * 5).astype(np.float32)
    y = (rng.integers(0, H // 5, n) * 5).astype(np.float32)
    x[:40], y[40:80] = 0.0, float(H - 1)
    k = _kps(x, y, rng.integers(0, 3, n))
    d = random_descriptors(n, 14)
    nq = 4000
    src = rng.integers(0, n, nq)   # centred up to a cell from a feature, so edge features put windows past the edges
    qu = (x[src] + rng.integers(-2, 3, nq) * 5).astype(np.float32)
    qv = (y[src] + rng.integers(-2, 3, nq) * 5).astype(np.float32)
    qr = rng.choice(np.array([2.5, 5.0, 10.0, 15.0, 20.0], np.float32), nq)
    qd = noisy_copies(d[src], 0.1, 15)
    v, o = _views(k, d)
    m = fe.ORBmatcher(0.8, False)
    got = _same(m, v, o, qu, qv, qr, np.full(nq, -1, np.int32), np.full(nq, -1, np.int32), qd, 100)
    assert (got >= 0).sum() > 1000
    m.close()


@pytest.mark.gpu
@pytest.mark.parametrize("force_scratch", [False, True])
def test_more_queries_than_one_launch(gpu_required, monkeypatch, force_scratch):
    """30000 queries into a 2000-feature frame need two launches; the result equals the oracle's single loop, with the
    candidate entries in shared memory or all in the global scratch."""
    if force_scratch:
        monkeypatch.setenv("ORBFE_SBP_FORCE_SCRATCH", "1")
    k, d, qu, qv, qr, lo, hi, qd = _random_scene(2000, 30000, seed=21, r=(3.0, 24.0))
    v, o = _views(k, d)
    m = fe.ORBmatcher(0.8, False)
    for nq, launches in ((LIMIT, 1), (30000, 2)):
        n0 = m.counters()[2]
        got = _same(m, v, o, qu[:nq], qv[:nq], qr[:nq], lo[:nq], hi[:nq], qd[:nq], 50)
        assert m.counters()[2] - n0 == launches and (got >= 0).sum() > nq // 6
    m.close()


@pytest.mark.gpu
@pytest.mark.parametrize("rule", [0, 1, 2])
def test_guided_search_above_one_launch(gpu_required, rule):
    """orbfe_guided_search without the rotation histogram past the single-launch limit: consecutive launches against the
    same slots equal the oracle's loop (later queries lose slots that earlier launches took; occupied slots stay), and just
    below the limit the call is one launch with the same answer.  With the histogram (hist_mode 1) the call is refused."""
    k, d, qu, qv, qr, lo, hi, qd = _random_scene(2000, 30000, seed=30 + rule, r=(3.0, 24.0))
    ang = np.random.default_rng(40).uniform(0, 360, 30000).astype(np.float32)
    occ = np.full(2000, -1, np.int32)
    occ[np.random.default_rng(41).random(2000) < 0.05] = 7
    v, o = _views(k, d)
    m = fe.ORBmatcher(0.8, False)
    for nq, launches in ((LIMIT, 1), (30000, 2)):
        for hist in (0, 2):
            n0 = m.counters()[2]
            n, so = M.guided_search(m, v, qu[:nq], qv[:nq], qr[:nq], lo[:nq], hi[:nq], qd[:nq], ang[:nq], rule, 64, hist, slot_owner=occ)
            n_o, so_o = O.guided_search(o, qu[:nq], qv[:nq], qr[:nq], lo[:nq], hi[:nq], qd[:nq], ang[:nq], rule, 0.8, 64, hist,
                                        slot_owner=occ)
            assert n == n_o > 200 and np.array_equal(so, so_o), (nq, hist)
            assert m.counters()[2] - n0 == launches
            assert nq == LIMIT or (so >= LIMIT).sum() > 20   # slots taken by queries of the second launch
    with pytest.raises(fe.OrbfeError) as e:
        M.guided_search(m, v, qu, qv, qr, lo, hi, qd, ang, rule, 64, 1, slot_owner=occ)
    assert e.value.code == fe.ORBFE_ERR_UNSUPPORTED and "220 KB" in str(e.value)
    m.close()
